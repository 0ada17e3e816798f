// msm_k_pair.cuh — batched-affine pair-add kernel and its launcher.
#pragma once
#include "msm_common.cuh"

namespace ab200 {

template <class F, bool FIRST>
__device__ __forceinline__ void pair_load_point(uint32_t *x, uint32_t *y, const uint32_t *__restrict__ bases, const uint32_t *__restrict__ src,
                                                uint32_t k) {
    constexpr int L = F::L;
    if (FIRST) {
        const uint32_t e = __ldg(src + k);
        const uint32_t *bp = bases + (size_t)(e & 0x7fffffffu) * (2 * L);
        load_limbs_nc<L>(x, bp);
        load_limbs_nc<L>(y, bp + L);
        F::cneg(y, y, (e >> 31) != 0);   // -(0,0) stays (0,0)
    } else {
        const uint32_t *bp = src + (size_t)k * (2 * L);
        load_limbs_nc<L>(x, bp);
        load_limbs_nc<L>(y, bp + L);
    }
}

enum { PAIR_PASS1 = 0, PAIR_PASS2 = 1, PAIR_INF = 2, PAIR_ADD = 3, PAIR_DBL = 4 };
// classify (P1, P2) and produce the denominator of the slope (ONE for the degenerate kinds)
template <class F> __device__ __forceinline__ int pair_classify(uint32_t *den, const uint32_t *x1, const uint32_t *y1, const uint32_t *x2,
                                                                const uint32_t *y2, bool has2) {
    constexpr int L = F::L;
    const bool z1 = limbs_is_zero<L>(x1) && limbs_is_zero<L>(y1);
    const bool z2 = !has2 || (limbs_is_zero<L>(x2) && limbs_is_zero<L>(y2));
    F::set_one(den);
    if (z2) return PAIR_PASS1;            // also covers "both identity" (P1 = (0,0) passes through)
    if (z1) return PAIR_PASS2;
    if (limbs_eq<L>(x1, x2)) {
        if (limbs_eq<L>(y1, y2) && !limbs_is_zero<L>(y1)) { F::dbl(den, y1); return PAIR_DBL; }
        return PAIR_INF;
    }
    F::sub(den, x2, x1);
    return PAIR_ADD;
}


// Inverts the 128 per-thread products of a block with ONE field inversion (Montgomery's trick across the block): warp 0 takes
// 4 products per lane, combines the 32 lane totals with a shuffle scan (prefix and suffix products), inverts the grand total and
// peels the 128 inverses back out; every thread then picks up 1/run of its own product.  A per-thread inversion costs ~570
// multiplications of issue time PER WARP; this costs ~590 per BLOCK, i.e. a quarter — which is what allows short batches.
// `sm` holds 128 * L words (word i of thread t at sm[i * 128 + t]); all 128 threads of the block must call this.
// The inversion is the plain square-and-multiply F::inv, not Fp::inv_lowlat (4-bit windows + symmetric squaring): the latter's
// table lives in local memory and sqr_sos has more carry-ripple adds than mul(a, a).
template <class F> __device__ __forceinline__ void shfl_limbs(uint32_t *r, const uint32_t *a, int src_lane) {
#pragma unroll
    for (int i = 0; i < F::L; i++) r[i] = __shfl_sync(0xffffffffu, a[i], src_lane);
}
template <class F> __device__ __noinline__ void block_inverse(uint32_t *inv, const uint32_t *run, uint32_t *sm) {
    constexpr int L = F::L;
    const int tid = threadIdx.x, lane = tid & 31;
    __syncthreads();   // `sm` may alias staging strips that slower warps of the block are still reading
#pragma unroll
    for (int i = 0; i < L; i++) sm[i * 128 + tid] = run[i];
    __syncthreads();
    if (tid < 32) {
        auto rd = [&](uint32_t *v, int j) {
#pragma unroll
            for (int i = 0; i < L; i++) v[i] = sm[i * 128 + 4 * lane + j];
        };
        auto wr = [&](const uint32_t *v, int j) {
#pragma unroll
            for (int i = 0; i < L; i++) sm[i * 128 + 4 * lane + j] = v[i];
        };
        uint32_t v[L], a1[L], a2[L], a3[L], P[L], S[L], y[L];
        rd(a1, 0); rd(v, 1); F::mul(a1, a1, v);      // a1 = v0 v1
        rd(v, 2); F::mul(a2, a1, v);                 // a2 = v0 v1 v2
        rd(v, 3); F::mul(a3, a2, v);                 // a3 = lane total
        limbs_copy<L>(P, a3);
        limbs_copy<L>(S, a3);
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {           // inclusive prefix (P) and suffix (S) products over the lanes
            shfl_limbs<F>(y, P, lane >= o ? lane - o : lane);
            if (lane >= o) F::mul(P, P, y);
            shfl_limbs<F>(y, S, lane + o < 32 ? lane + o : lane);
            if (lane + o < 32) F::mul(S, S, y);
        }
        uint32_t I[L];
        shfl_limbs<F>(y, P, 31);
        F::inv(I, y);                                 // 1 / (product of all 128), computed redundantly by the 32 lanes
        shfl_limbs<F>(y, P, lane ? lane - 1 : 0);
        if (lane) F::mul(I, I, y);                    // ... times the products of the other lanes = 1 / a3
        shfl_limbs<F>(y, S, lane < 31 ? lane + 1 : 31);
        if (lane < 31) F::mul(I, I, y);
        // peel: I = 1/(v0 v1 v2 v3)
        rd(v, 3); F::mul(y, I, a2); F::mul(I, I, v); wr(y, 3);     // 1/v3 = I a2 ; I <- 1/(v0 v1 v2)
        rd(v, 2); F::mul(y, I, a1); F::mul(I, I, v); wr(y, 2);     // 1/v2 = I a1 ; I <- 1/(v0 v1)
        rd(v, 1); rd(a1, 0);
        F::mul(y, I, a1); wr(y, 1);                                  // 1/v1 = I v0
        F::mul(y, I, v); wr(y, 0);                                   // 1/v0 = I v1
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < L; i++) inv[i] = sm[i * 128 + tid];
    __syncthreads();   // `sm` may be reused by the caller (the staging strips of the pair-add kernel)
}

// ------------------------------------------------------------------------------------------------
// Pair-add: warp-interleaved slots + asynchronous operand staging.
//   * a WARP owns 32*batch consecutive output slots and lane l takes slots l, l+32, l+64, ... — every Montgomery-trick chain is
//     still private to one thread, but the 32 lanes of a load/store touch 32 consecutive slots (coalesced streaming for the
//     levels >= 2 and for the parked prefix products);
//   * the operands of the NEXT slot are fetched with cp.async (LDGSTS) into a per-thread shared-memory strip while the current
//     slot's multiplications run, so the random 96-byte gathers of level 1 do not stall the integer pipe and cost no registers;
//   * slot -> input-pair mapping comes from `pairmap` (msm_pairmap_kernel);
//   * the running products of the 128 threads of a block share one field inversion (block_inverse).
// ------------------------------------------------------------------------------------------------
// cp.async.ca allocates in L1: the three 16-byte chunks of a 48-byte coordinate, and x then y of a point, hit the line the first
// chunk brought in
__device__ __forceinline__ void cp_async16(uint32_t saddr, const void *g) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(saddr), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// per-thread strip: element e, 16-byte chunk j of thread t lives at uint4 index (e*(L/4) + j)*128 + t (conflict-free)
template <int L> __device__ __forceinline__ void strip_fetch(uint32_t sbase, int e, const uint32_t *g) {
#pragma unroll
    for (int j = 0; j < L / 4; j++) cp_async16(sbase + ((uint32_t)((e * (L / 4) + j) * 128 + threadIdx.x) << 4), g + 4 * j);
}
template <int L> __device__ __forceinline__ void strip_read(uint32_t *r, const uint4 *sm, int e) {
#pragma unroll
    for (int j = 0; j < L / 4; j++) {
        const uint4 v = sm[(e * (L / 4) + j) * 128 + threadIdx.x];
        r[4 * j] = v.x; r[4 * j + 1] = v.y; r[4 * j + 2] = v.z; r[4 * j + 3] = v.w;
    }
}

template <class C, bool FIRST>
__global__ void __launch_bounds__(128, C::PAIR_MINB) msm_pair_add_kernel(const uint32_t *__restrict__ bases, const uint32_t *__restrict__ src,
                                                                        const uint32_t *__restrict__ pairmap, const uint32_t *__restrict__ offsets_out,
                                                                        uint32_t nb, uint32_t batch, uint32_t *__restrict__ out) {
    using F = typename C::F;
    constexpr int L = F::L;
    extern __shared__ uint4 strip[];
    const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(strip);
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t M = __ldg(offsets_out + nb);
    const uint64_t w_lo = (uint64_t)blockIdx.x * 128 * batch + (uint64_t)(threadIdx.x >> 5) * 32 * batch;
    // a lane without slots still runs to block_inverse: every thread of the block has to reach its barriers
    const bool active = w_lo + lane < M;
    const uint32_t w_hi = (uint32_t)min((uint64_t)M, w_lo + (uint64_t)32 * batch);
    const uint32_t p0 = active ? (uint32_t)w_lo + lane : 0;
    const uint32_t cnt = active ? (w_hi - p0 + 31) >> 5 : 0;   // slots p0 + 32*i, i < cnt
    // address of the point behind input entry `k` (FIRST: through the sorted index, e = index | sign << 31)
    auto point = [&](uint32_t k, uint32_t e) -> const uint32_t * {
        return FIRST ? bases + (size_t)(e & 0x7fffffffu) * (2 * L) : src + (size_t)k * (2 * L);
    };
    uint32_t x1[L], y1[L], x2[L], y2[L], den[L], run[L];
    // software pipeline over the slots of this lane: (m, e1, e2) describe a slot (pairmap word and, for FIRST, the two sorted
    // entries); *_c = slot being computed, *_n = next slot (operands in flight), m_nn = pairmap word two slots ahead
    uint32_t m_c, m_n = 0, m_nn = 0, e1_c = 0, e2_c = 0, e1_n = 0, e2_n = 0;

    // ---------------- forward: running product of the denominators (x coordinates only), parked in the x-half of the slots
    F::set_one(run);
    if (cnt) {
    m_c = __ldg(pairmap + p0);
    if (FIRST) { e1_c = __ldg(src + (m_c & 0x7fffffffu)); if (m_c >> 31) e2_c = __ldg(src + (m_c & 0x7fffffffu) + 1); }
    // (forward uses strip elements {0,2} for even slots and {1,3} for odd ones: a true double buffer)
    if (m_c >> 31) { strip_fetch<L>(sbase, 0, point(m_c & 0x7fffffffu, e1_c)); strip_fetch<L>(sbase, 2, point((m_c & 0x7fffffffu) + 1, e2_c)); }
    cp_async_commit();
    if (cnt > 1) {
        m_n = __ldg(pairmap + p0 + 32);
        if (FIRST) { e1_n = __ldg(src + (m_n & 0x7fffffffu)); if (m_n >> 31) e2_n = __ldg(src + (m_n & 0x7fffffffu) + 1); }
    }
    if (cnt > 2) m_nn = __ldg(pairmap + p0 + 64);
    for (uint32_t i = 0; i < cnt; i++) {
        cp_async_wait_all();
        const bool has2 = (m_c >> 31) != 0;
        const int eb = (int)(i & 1);
        if (has2) { strip_read<L>(x1, strip, eb); strip_read<L>(x2, strip, 2 + eb); }
        if (i + 1 < cnt && (m_n >> 31)) {
            strip_fetch<L>(sbase, 1 - eb, point(m_n & 0x7fffffffu, e1_n));
            strip_fetch<L>(sbase, 3 - eb, point((m_n & 0x7fffffffu) + 1, e2_n));
        }
        cp_async_commit();
        uint32_t e1_nn = 0, e2_nn = 0, m_n3 = 0;
        if (FIRST && i + 2 < cnt) { e1_nn = __ldg(src + (m_nn & 0x7fffffffu)); if (m_nn >> 31) e2_nn = __ldg(src + (m_nn & 0x7fffffffu) + 1); }
        if (i + 3 < cnt) m_n3 = __ldg(pairmap + p0 + 32 * (i + 3));
        if (has2) {
            if (limbs_is_zero<L>(x1) || limbs_is_zero<L>(x2) || limbs_eq<L>(x1, x2)) {   // rare: identity operand / equal x
                const uint32_t k = m_c & 0x7fffffffu;
                pair_load_point<F, FIRST>(x1, y1, bases, src, k);
                pair_load_point<F, FIRST>(x2, y2, bases, src, k + 1);
                const int kind = pair_classify<F>(den, x1, y1, x2, y2, true);
                if (kind >= PAIR_ADD) F::mul(run, run, den);
            } else {
                F::sub(den, x2, x1);
                F::mul(run, run, den);
            }
        }
        store_limbs<L>(out + (size_t)(p0 + 32 * i) * (2 * L), run);
        m_c = m_n; e1_c = e1_n; e2_c = e2_n;
        m_n = m_nn; e1_n = e1_nn; e2_n = e2_nn;
        m_nn = m_n3;
    }
    }
    uint32_t inv[L];
    block_inverse<F>(inv, run, reinterpret_cast<uint32_t *>(strip));   // (no copy is in flight here: the strips are free)
    if (!cnt) return;

    // ---------------- backward: peel the inverses off and write the sums; strip elements 0..3 = x1, y1, x2, y2, 4 = prefix
    auto fetch_bwd = [&](uint32_t m, uint32_t e1, uint32_t e2, uint32_t i) {   // operands of slot i and the prefix parked in slot i-1
        const uint32_t k = m & 0x7fffffffu;
        const uint32_t *a = point(k, e1);
        strip_fetch<L>(sbase, 0, a);
        strip_fetch<L>(sbase, 1, a + L);
        if (m >> 31) {
            const uint32_t *b = point(k + 1, e2);
            strip_fetch<L>(sbase, 2, b);
            strip_fetch<L>(sbase, 3, b + L);
        }
        if (i > 0) strip_fetch<L>(sbase, 4, out + (size_t)(p0 + 32 * (i - 1)) * (2 * L));
    };
    m_c = __ldg(pairmap + p0 + 32 * (cnt - 1));
    e1_c = e2_c = e1_n = e2_n = 0;
    m_n = m_nn = 0;
    if (FIRST) { e1_c = __ldg(src + (m_c & 0x7fffffffu)); if (m_c >> 31) e2_c = __ldg(src + (m_c & 0x7fffffffu) + 1); }
    fetch_bwd(m_c, e1_c, e2_c, cnt - 1);
    cp_async_commit();
    if (cnt > 1) {
        m_n = __ldg(pairmap + p0 + 32 * (cnt - 2));
        if (FIRST) { e1_n = __ldg(src + (m_n & 0x7fffffffu)); if (m_n >> 31) e2_n = __ldg(src + (m_n & 0x7fffffffu) + 1); }
    }
    if (cnt > 2) m_nn = __ldg(pairmap + p0 + 32 * (cnt - 3));
    for (uint32_t i = cnt; i-- > 0;) {
        cp_async_wait_all();
        const bool has2 = (m_c >> 31) != 0;
        uint32_t dinv[L];
        strip_read<L>(x1, strip, 0);
        strip_read<L>(y1, strip, 1);
        if (has2) { strip_read<L>(x2, strip, 2); strip_read<L>(y2, strip, 3); }
        if (i > 0) { strip_read<L>(dinv, strip, 4); F::mul(dinv, inv, dinv); }   // inv * prefix_{i-1} = 1/den_i
        else limbs_copy<L>(dinv, inv);
        if (FIRST) {
            F::cneg(y1, y1, (e1_c >> 31) != 0);
            if (has2) F::cneg(y2, y2, (e2_c >> 31) != 0);
        }
        if (i > 0) fetch_bwd(m_n, e1_n, e2_n, i - 1);
        cp_async_commit();
        uint32_t e1_nn = 0, e2_nn = 0, m_n3 = 0;
        if (FIRST && i >= 2) { e1_nn = __ldg(src + (m_nn & 0x7fffffffu)); if (m_nn >> 31) e2_nn = __ldg(src + (m_nn & 0x7fffffffu) + 1); }
        if (i >= 3) m_n3 = __ldg(pairmap + p0 + 32 * (i - 3));
        const int kind = pair_classify<F>(den, x1, y1, x2, y2, has2);
        uint32_t *o = out + (size_t)(p0 + 32 * i) * (2 * L);
        if (kind >= PAIR_ADD) {
            uint32_t lam[L], t3[L];
            F::mul(inv, inv, den);
            if (kind == PAIR_ADD) {
                F::sub(lam, y2, y1);
            } else {                      // doubling: slope = 3 x^2 / (2 y)
                F::sqr(lam, x1);
                F::dbl(t3, lam);
                F::add(lam, lam, t3);
                limbs_copy<L>(x2, x1);
            }
            F::mul(lam, lam, dinv);
            F::sqr(t3, lam);
            F::sub(t3, t3, x1);
            F::sub(t3, t3, x2);           // x3
            F::sub(x2, x1, t3);
            F::mul(x2, lam, x2);
            F::sub(x2, x2, y1);           // y3 = lam (x1 - x3) - y1
            store_limbs<L>(o, t3);
            store_limbs<L>(o + L, x2);
        } else if (kind == PAIR_PASS1) {
            store_limbs<L>(o, x1);
            store_limbs<L>(o + L, y1);
        } else if (kind == PAIR_PASS2) {
            store_limbs<L>(o, x2);
            store_limbs<L>(o + L, y2);
        } else {
            F::set_zero(x1);
            store_limbs<L>(o, x1);
            store_limbs<L>(o + L, x1);
        }
        m_c = m_n; e1_c = e1_n; e2_c = e2_n;
        m_n = m_nn; e1_n = e1_nn; e2_n = e2_nn;
        m_nn = m_n3;
    }
}

template <class C>
int MsmPairLaunch<C>::run(bool first, const uint32_t *bases, const uint32_t *src, const uint32_t *offsets_out, const uint32_t *pairmap, uint32_t nbg,
                          uint32_t batch, size_t out_cap, uint32_t *out, cudaStream_t st) {
    constexpr int L = C::F::L;
    const size_t warps = (out_cap + (size_t)32 * batch - 1) / ((size_t)32 * batch);
    const unsigned pg = (unsigned)((warps + 3) / 4);
    const size_t smem = (size_t)5 * (L / 4) * 128 * 16;
    auto kernel = first ? msm_pair_add_kernel<C, true> : msm_pair_add_kernel<C, false>;
    AB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<pg, 128, smem, st>>>(bases, src, pairmap, offsets_out, nbg, batch, out);
    AB_LAUNCHED();
    return 0;
}

}  // namespace ab200
