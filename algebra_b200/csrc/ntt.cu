// ntt.cu — radix-2 NTT over a 4-limb (8 x u32) Montgomery scalar field, for sm_90a.
//
// Replaces Radix2EvaluationDomain::{fft_in_place, ifft_in_place} after the resize step
// (poly/src/domain/radix2/mod.rs:140-153 -> fft.rs:74-88: io_helper/oi_helper + derange + scaling).
// Field arithmetic is exact and every element is kept fully reduced, so any correct evaluation order is
// bit-identical to the reference's DIF+bit-reversal; this file uses a multi-pass decimation tuned for the GPU:
//
//   n = A_1 * A_2 * ... * A_m  (A_t = 2^{r_t} <= 256).  Pass t works inside contiguous segments of length
//   seg_t = n / (A_1..A_{t-1}):  with B = seg_t / A_t and j = a*B + b, i = iA + A_t*iB
//        w_seg^{ij} = w_A^{a*iA} * w_seg^{b*iA} * w_B^{b*iB}
//   so a pass is (1) an A_t-point NTT down each stride-B column, held in shared memory, (2) one multiplication
//   by the "segment twiddle" w_seg^{b*iA} (table laid out [iA][b] so it is read exactly like the data), stored in
//   place at row iA.  The last pass (B = 1) has no twiddle and writes each value to its final natural-order
//   index (digit reversal of the row indices), G adjacent outputs (G*32 B) at a time.
//   Pass 1 reads the user buffer and writes scratch, middle passes run in place on scratch, the last pass
//   writes back to the user buffer — no extra copy, natural order in and out.
//
// Work per element: sum_t r_t/2 butterfly multiplies (the gap-1 stage of every pass has w = 1 and is skipped)
// + (m-1) segment-twiddle multiplies.  2^24 = 256^3: 3*3.5 + 2 = 12.5 modmuls/element (136 IMAD.WIDE each).
// HBM traffic: m reads + m writes of the data + (m-1) table reads (L2-resident except the pass-1 table).
// 1/n of the inverse transform is folded into the pass-1 table; coset scaling is a separate element-wise kernel.
#include <map>
#include <memory>
#include <mutex>
#include <tuple>
#include <vector>

#include "common.cuh"
#include "host_api.h"

namespace ab200 {

static constexpr int kMaxLogRadix = 8;           // A <= 256
static constexpr int kSmallTabLog = kMaxLogRadix - 1;  // w_256^t for t < 128
static constexpr int kMaxPasses = 4;

struct NttPassParams {
    int log_n, r, logG, log_seg, is_last;
    int m, radix_log[kMaxPasses];  // all pass radices (last pass: digit reversal)
    const uint4 *tw_small;          // w_{256}^t, t < 128 (Montgomery), forward or inverse root
    const uint4 *tw_seg;            // [iA][b] segment twiddles of this pass, or nullptr
    int has_scale;                  // single-pass inverse: multiply by 1/n at the store
    uint32_t scale[8];
};

// shared-memory tile: two 16-byte planes so that consecutive elements are consecutive uint4 (conflict-free)
template <class P>
__global__ void __launch_bounds__(512, 2) ntt_pass_kernel(const uint4 *in, uint4 *out, NttPassParams pp) {
    using F = Fp<P>;
    extern __shared__ uint4 smem[];
    const int r = pp.r, logG = pp.logG, G = 1 << logG, A = 1 << r;
    const int tile = A << logG;           // elements in the tile
    uint4 *s_lo = smem, *s_hi = smem + tile;
    const int tid = threadIdx.x, nthreads = blockDim.x;  // == tile / 2 (or 1 when tile == 1.. never)
    const unsigned bid = blockIdx.x;
    const int logB = pp.log_seg - r;

    // ---- tile geometry
    size_t seg_base = 0;   // non-last: sigma * seg
    size_t b0 = 0;         // non-last: first column
    size_t g0 = 0, q = 0;  // last: first i1, and the (i2..i_{m-1}) index
    const int logA1 = pp.radix_log[0];
    if (!pp.is_last) {
        const int log_cg = logB - logG;  // column groups per segment
        seg_base = (size_t)(bid >> log_cg) << pp.log_seg;
        b0 = (size_t)(bid & ((1u << log_cg) - 1)) << logG;
    } else if (pp.m > 1) {
        const int log_i1g = logA1 - logG;
        g0 = (size_t)(bid & ((1u << log_i1g) - 1)) << logG;
        q = bid >> log_i1g;
    }

    // ---- load (2 elements per thread)
#pragma unroll
    for (int k = 0; k < 2; k++) {
        int idx = tid + k * nthreads;
        if (idx < tile) {
            size_t pos;
            int sidx;
            if (!pp.is_last) {
                int a = idx >> logG, g = idx & (G - 1);
                pos = seg_base + ((size_t)a << logB) + b0 + g;
                sidx = idx;
            } else {
                int g = idx >> r, a = idx & (A - 1);
                pos = (pp.m > 1) ? (((g0 + g) << (pp.log_n - logA1)) + (q << r) + a) : (size_t)a;
                sidx = (a << logG) + g;
            }
            s_lo[sidx] = in[2 * pos];
            s_hi[sidx] = in[2 * pos + 1];
        }
    }
    __syncthreads();

    // ---- r DIF stages: lo' = lo + hi ; hi' = (lo - hi) * w     (butterfly_fn_io, fft.rs:190-198)
    // The last two stages (gaps 2 and 1) are fused into one radix-4 step on 4 consecutive rows held in registers: three of its four
    // butterflies have w = 1, so it costs ONE twiddle multiplication (by the 4th root of unity) per 4 elements instead of two, and
    // saves a barrier and a shared-memory round trip.
    {
        const bool active = tid < tile / 2;
        const int g = tid & (G - 1), u = tid >> logG;
        const int radix2_stages = r >= 2 ? r - 2 : r;
        for (int s = 0; s < radix2_stages; s++) {
            if (active) {
                const int gaplog = r - 1 - s;
                const int j = u & ((1 << gaplog) - 1);
                const int lo_a = ((u >> gaplog) << (gaplog + 1)) | j;
                const int li = (lo_a << logG) + g, hi = li + ((1 << gaplog) << logG);
                uint32_t x[8], y[8], d[8];
                uint4 t0 = s_lo[li], t1 = s_hi[li], t2 = s_lo[hi], t3 = s_hi[hi];
                x[0] = t0.x; x[1] = t0.y; x[2] = t0.z; x[3] = t0.w; x[4] = t1.x; x[5] = t1.y; x[6] = t1.z; x[7] = t1.w;
                y[0] = t2.x; y[1] = t2.y; y[2] = t2.z; y[3] = t2.w; y[4] = t3.x; y[5] = t3.y; y[6] = t3.z; y[7] = t3.w;
                F::sub(d, x, y);
                F::add(x, x, y);
                if (gaplog != 0) {  // the gap-1 stage only has w = 1
                    uint32_t w[8];
                    const uint4 *tw = pp.tw_small + 2 * ((size_t)(j << s) << (kMaxLogRadix - r));
                    uint4 w0 = __ldg(tw), w1 = __ldg(tw + 1);
                    w[0] = w0.x; w[1] = w0.y; w[2] = w0.z; w[3] = w0.w; w[4] = w1.x; w[5] = w1.y; w[6] = w1.z; w[7] = w1.w;
                    F::mul(d, d, w);
                }
                s_lo[li] = make_uint4(x[0], x[1], x[2], x[3]);
                s_hi[li] = make_uint4(x[4], x[5], x[6], x[7]);
                s_lo[hi] = make_uint4(d[0], d[1], d[2], d[3]);
                s_hi[hi] = make_uint4(d[4], d[5], d[6], d[7]);
            }
            __syncthreads();
        }
        if (r >= 2) {
            if (tid < tile / 4) {   // group (q, g): rows 4q .. 4q+3 of column g
                const int q = tid >> logG, base = ((4 * q) << logG) + g;
                uint32_t x[4][8], t[8], w[8];
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    const uint4 a = s_lo[base + (e << logG)], b = s_hi[base + (e << logG)];
                    x[e][0] = a.x; x[e][1] = a.y; x[e][2] = a.z; x[e][3] = a.w; x[e][4] = b.x; x[e][5] = b.y; x[e][6] = b.z; x[e][7] = b.w;
                }
                F::sub(t, x[0], x[2]); F::add(x[0], x[0], x[2]); limbs_copy<8>(x[2], t);          // gap 2, j = 0: w = 1
                F::sub(t, x[1], x[3]); F::add(x[1], x[1], x[3]);                                  // gap 2, j = 1: w = w_4 = w_256^64
                {
                    const uint4 w0 = __ldg(pp.tw_small + 2 * 64), w1 = __ldg(pp.tw_small + 2 * 64 + 1);
                    w[0] = w0.x; w[1] = w0.y; w[2] = w0.z; w[3] = w0.w; w[4] = w1.x; w[5] = w1.y; w[6] = w1.z; w[7] = w1.w;
                }
                F::mul(x[3], t, w);
                F::sub(t, x[0], x[1]); F::add(x[0], x[0], x[1]); limbs_copy<8>(x[1], t);          // gap 1
                F::sub(t, x[2], x[3]); F::add(x[2], x[2], x[3]); limbs_copy<8>(x[3], t);
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    s_lo[base + (e << logG)] = make_uint4(x[e][0], x[e][1], x[e][2], x[e][3]);
                    s_hi[base + (e << logG)] = make_uint4(x[e][4], x[e][5], x[e][6], x[e][7]);
                }
            }
            __syncthreads();
        }
    }

    // ---- store: smem row t holds sub-NTT output iA = bitrev_r(t)
#pragma unroll
    for (int k = 0; k < 2; k++) {
        int idx = tid + k * nthreads;
        if (idx < tile) {
            const int t = idx >> logG, g = idx & (G - 1);
            const size_t iA = r ? (__brev((unsigned)t) >> (32 - r)) : 0;
            uint4 v0 = s_lo[idx], v1 = s_hi[idx];
            size_t pos;
            if (!pp.is_last) {
                const size_t off = (iA << logB) + b0 + g;
                pos = seg_base + off;
                uint32_t v[8], w[8];
                uint4 w0 = __ldg(pp.tw_seg + 2 * off), w1 = __ldg(pp.tw_seg + 2 * off + 1);
                v[0] = v0.x; v[1] = v0.y; v[2] = v0.z; v[3] = v0.w; v[4] = v1.x; v[5] = v1.y; v[6] = v1.z; v[7] = v1.w;
                w[0] = w0.x; w[1] = w0.y; w[2] = w0.z; w[3] = w0.w; w[4] = w1.x; w[5] = w1.y; w[6] = w1.z; w[7] = w1.w;
                F::mul(v, v, w);
                v0 = make_uint4(v[0], v[1], v[2], v[3]);
                v1 = make_uint4(v[4], v[5], v[6], v[7]);
            } else {
                if (pp.has_scale) {
                    uint32_t v[8];
                    v[0] = v0.x; v[1] = v0.y; v[2] = v0.z; v[3] = v0.w; v[4] = v1.x; v[5] = v1.y; v[6] = v1.z; v[7] = v1.w;
                    F::mul(v, v, pp.scale);
                    v0 = make_uint4(v[0], v[1], v[2], v[3]);
                    v1 = make_uint4(v[4], v[5], v[6], v[7]);
                }
                if (pp.m > 1) {
                    // position digits (i1 | i2 .. i_{m-1} | i_m)  ->  index i1 + A1*(i2 + A2*(... + A_{m-1}*i_m))
                    size_t rev = 0, rem = q;
                    int shift = 0, pv = pp.log_n - logA1 - r;  // log of the number of q values
                    for (int d = 1; d < pp.m - 1; d++) {
                        pv -= pp.radix_log[d];
                        rev += (rem >> pv) << shift;
                        rem &= ((size_t)1 << pv) - 1;
                        shift += pp.radix_log[d];
                    }
                    pos = (g0 + g) + ((rev + (iA << shift)) << logA1);
                } else {
                    pos = iA;
                }
            }
            out[2 * pos] = v0;
            out[2 * pos + 1] = v1;
        }
    }
}

// tab[iA*B + b] = scale * w^(iA*b), iA < A, b < B; one thread per (iA, 16 consecutive b)
template <class P>
__global__ void gen_seg_twiddles_kernel(uint4 *tab, LimbArg<8> w, LimbArg<8> scale, int logA, int logB) {
    using F = Fp<P>;
    const int CH = 16;
    size_t gid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t B = (size_t)1 << logB;
    size_t chunks_per_row = (B + CH - 1) / CH;
    size_t iA = gid / chunks_per_row, bstart = (gid % chunks_per_row) * CH;
    if (iA >= ((size_t)1 << logA)) return;
    uint32_t base[8], cur[8];
    F::pow_u64(base, w.v, iA);
    F::pow_u64(cur, base, bstart);
    F::mul(cur, cur, scale.v);
    for (size_t b = bstart; b < bstart + CH && b < B; b++) {
        size_t o = (iA << logB) + b;
        tab[2 * o] = make_uint4(cur[0], cur[1], cur[2], cur[3]);
        tab[2 * o + 1] = make_uint4(cur[4], cur[5], cur[6], cur[7]);
        F::mul(cur, cur, base);
    }
}

// x[i] *= c * g^i   (distribute_powers_and_mul_by_const, poly/src/domain/mod.rs:119-148); 16 elements per thread
template <class P> __global__ void distribute_powers_kernel(uint4 *x, size_t n, LimbArg<8> g, LimbArg<8> c) {
    using F = Fp<P>;
    const int CH = 16;
    size_t i0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * CH;
    if (i0 >= n) return;
    uint32_t pw[8];
    F::pow_u64(pw, g.v, i0);
    F::mul(pw, pw, c.v);
    for (size_t i = i0; i < i0 + CH && i < n; i++) {
        uint4 v0 = x[2 * i], v1 = x[2 * i + 1];
        uint32_t v[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
        F::mul(v, v, pw);
        x[2 * i] = make_uint4(v[0], v[1], v[2], v[3]);
        x[2 * i + 1] = make_uint4(v[4], v[5], v[6], v[7]);
        F::mul(pw, pw, g.v);
    }
}

// ------------------------------------------------------------------------------------------------
// host side: plans (twiddle tables) cached per (device, field, log_n, direction)
// ------------------------------------------------------------------------------------------------
struct NttPlan {
    int log_n = 0, m = 0;
    int radix_log[kMaxPasses] = {0, 0, 0, 0};
    uint4 *tw_small = nullptr;
    uint4 *tw_seg[kMaxPasses] = {nullptr, nullptr, nullptr, nullptr};
    uint32_t scale[8];  // 1/n (Montgomery) for the inverse, ONE otherwise
    bool inverse = false;
};
// Plans are shared_ptr-owned: a transform keeps its plan alive while it runs, so a concurrent b200_clear_cache (or an LRU eviction)
// only drops the cache's reference; the tables are freed when the last user lets go (cudaFree waits for kernels still reading them).
// The cache is bounded: least-recently-used plans are evicted once the cached tables exceed kPlanCacheBytes.
struct NttPlanOwner {
    NttPlan p;
    size_t bytes = 0;
    uint64_t last_use = 0;
    ~NttPlanOwner();
};
static constexpr size_t kPlanCacheBytes = (size_t)6 << 30;
static std::mutex g_plan_mutex;
static std::map<std::tuple<int, int, int, int>, std::shared_ptr<NttPlanOwner>> g_plans;
static uint64_t g_plan_clock = 0;

template <class P> static void host_root_of_unity(uint32_t *g, int log_n) {
    // get_root_of_unity, ff/src/fields/fft_friendly.rs:66-82
    using F = Fp<P>;
    for (int i = 0; i < 8; i++) g[i] = P::TWO_ADIC_ROOT(i);
    for (int i = log_n; i < P::TWO_ADICITY; i++) F::sqr(g, g);
}

static void split_radices(int log_n, int &m, int *rl) {
    m = (log_n + kMaxLogRadix - 1) / kMaxLogRadix;
    if (m < 1) m = 1;
    int base = log_n / m, extra = log_n % m;
    for (int t = 0; t < m; t++) rl[t] = base + (t < extra ? 1 : 0);  // larger radices first
}

template <class P> static int build_plan(NttPlan &pl, int log_n, bool inverse, cudaStream_t st) {
    using F = Fp<P>;
    pl.log_n = log_n;
    pl.inverse = inverse;
    split_radices(log_n, pl.m, pl.radix_log);
    uint32_t g[8];
    host_root_of_unity<P>(g, log_n);
    if (inverse) F::inv(g, g);
    F::set_one(pl.scale);
    if (inverse) {  // size_inv (radix2/mod.rs:74)
        uint32_t nn[8] = {0};
        uint64_t n = (uint64_t)1 << log_n;
        nn[0] = (uint32_t)n;
        nn[1] = (uint32_t)(n >> 32);
        F::to_mont(nn, nn);
        F::inv(pl.scale, nn);
    }
    // small table: w_256^t, t < 128, with w_256 = g^(n/256) (or the primitive 2^log_n-th root padded when n < 256:
    // the kernel indexes it as w_A^t = w_256^(t * 256/A), so generate it from the 256-th root in this direction)
    {
        uint32_t w256[8];
        host_root_of_unity<P>(w256, kMaxLogRadix);
        if (inverse) F::inv(w256, w256);
        std::vector<uint32_t> tab((size_t)8 << kSmallTabLog);
        uint32_t cur[8];
        F::set_one(cur);
        for (int t = 0; t < (1 << kSmallTabLog); t++) {
            for (int i = 0; i < 8; i++) tab[8 * t + i] = cur[i];
            F::mul(cur, cur, w256);
        }
        AB_CUDA(cudaMalloc(&pl.tw_small, tab.size() * 4));
        AB_CUDA(cudaMemcpyAsync(pl.tw_small, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice, st));
        AB_CUDA(cudaStreamSynchronize(st));
    }
    // segment twiddles for every non-last pass
    int log_seg = log_n;
    for (int t = 0; t + 1 < pl.m; t++) {
        const int r = pl.radix_log[t], logB = log_seg - r;
        uint32_t wseg[8];  // w_seg = g^(n/seg)
        for (int i = 0; i < 8; i++) wseg[i] = g[i];
        for (int i = log_seg; i < log_n; i++) F::sqr(wseg, wseg);
        AB_CUDA(cudaMalloc(&pl.tw_seg[t], ((size_t)32) << log_seg));
        LimbArg<8> wa, sc;
        for (int i = 0; i < 8; i++) {
            wa.v[i] = wseg[i];
            sc.v[i] = (t == 0) ? pl.scale[i] : P::ONE(i);
        }
        size_t B = (size_t)1 << logB, chunks = (B + 15) / 16, threads = chunks << r;
        gen_seg_twiddles_kernel<P><<<(unsigned)((threads + 127) / 128), 128, 0, st>>>(pl.tw_seg[t], wa, sc, r, logB);
        AB_LAUNCHED();
        log_seg = logB;
    }
    AB_CUDA(cudaStreamSynchronize(st));
    return 0;
}

static void free_plan(NttPlan &pl) {
    if (pl.tw_small) cudaFree(pl.tw_small);
    for (auto &p : pl.tw_seg)
        if (p) cudaFree(p);
}
NttPlanOwner::~NttPlanOwner() { free_plan(p); }

int ntt_clear_cache() {
    std::vector<std::shared_ptr<NttPlanOwner>> dropped;   // destroyed (and their tables freed) outside the lock
    {
        std::lock_guard<std::mutex> lk(g_plan_mutex);
        int dev = 0;
        cudaGetDevice(&dev);
        for (auto it = g_plans.begin(); it != g_plans.end();) {
            if (std::get<0>(it->first) == dev) {
                dropped.push_back(it->second);
                it = g_plans.erase(it);
            } else ++it;
        }
    }
    return 0;
}

template <class P> static int ntt_run(int field, uint4 *d_data, int log_n, bool inverse, const uint64_t *coset, cudaStream_t st) {
    using F = Fp<P>;
    if (log_n > P::TWO_ADICITY) {
        set_last_error("log_n exceeds TWO_ADICITY (Radix2EvaluationDomain::new would return None)");
        return B200_ETOOLARGE;
    }
    const size_t n = (size_t)1 << log_n;
    uint32_t off[8];
    bool has_coset = false;
    if (coset) {
        for (int i = 0; i < 4; i++) {
            off[2 * i] = (uint32_t)coset[i];
            off[2 * i + 1] = (uint32_t)(coset[i] >> 32);
        }
        uint32_t one[8];
        F::set_one(one);
        has_coset = !limbs_eq<8>(off, one);  // `if !self.offset.is_one()` fft.rs:75
    }
    if (log_n == 0) return 0;  // size-1 domain: identity in both directions (size_inv = 1; offset^0 = 1)

    int dev = 0;
    AB_CUDA(cudaGetDevice(&dev));
    std::shared_ptr<NttPlanOwner> owner;   // keeps the tables alive for the duration of this transform
    std::vector<std::shared_ptr<NttPlanOwner>> evicted;
    {
        std::lock_guard<std::mutex> lk(g_plan_mutex);
        auto key = std::make_tuple(dev, field, log_n, (int)inverse);
        auto it = g_plans.find(key);
        if (it == g_plans.end()) {
            auto fresh = std::make_shared<NttPlanOwner>();
            int rc = build_plan<P>(fresh->p, log_n, inverse, st);
            if (rc) return rc;
            int ls = log_n;
            for (int t = 0; t + 1 < fresh->p.m; t++) { fresh->bytes += (size_t)32 << ls; ls -= fresh->p.radix_log[t]; }
            it = g_plans.emplace(key, fresh).first;
            size_t total = 0;
            for (auto &kv : g_plans) total += kv.second->bytes;
            while (total > kPlanCacheBytes && g_plans.size() > 1) {   // evict least recently used (never the one just built)
                auto victim = g_plans.end();
                for (auto jt = g_plans.begin(); jt != g_plans.end(); ++jt)
                    if (jt != it && (victim == g_plans.end() || jt->second->last_use < victim->second->last_use)) victim = jt;
                if (victim == g_plans.end()) break;
                total -= victim->second->bytes;
                evicted.push_back(victim->second);
                g_plans.erase(victim);
            }
        }
        owner = it->second;
        owner->last_use = ++g_plan_clock;
    }
    const NttPlan &plan = owner->p;
    LimbArg<8> one_arg, g_arg;
    for (int i = 0; i < 8; i++) one_arg.v[i] = P::ONE(i);

    if (has_coset && !inverse) {  // distribute_powers(x, offset), fft.rs:75-77
        for (int i = 0; i < 8; i++) g_arg.v[i] = off[i];
        size_t threads = (n + 15) / 16;
        distribute_powers_kernel<P><<<(unsigned)((threads + 127) / 128), 128, 0, st>>>(d_data, n, g_arg, one_arg);
        AB_LAUNCHED();
    }

    uint4 *scratch = nullptr;
    if (plan.m > 1) AB_CUDA(cudaMallocAsync(&scratch, n * 32, st));
    int log_seg = log_n;
    for (int t = 0; t < plan.m; t++) {
        NttPassParams pp;
        pp.log_n = log_n;
        pp.r = plan.radix_log[t];
        pp.log_seg = log_seg;
        pp.is_last = (t == plan.m - 1);
        pp.m = plan.m;
        for (int i = 0; i < kMaxPasses; i++) pp.radix_log[i] = plan.radix_log[i];
        pp.tw_small = plan.tw_small;
        pp.tw_seg = plan.tw_seg[t];
        pp.has_scale = (plan.m == 1 && inverse) ? 1 : 0;
        for (int i = 0; i < 8; i++) pp.scale[i] = plan.scale[i];
        const int logB = log_seg - pp.r;
        // G adjacent columns per block.  Small blocks (128-256 threads, 8-16 KB smem) keep ~10 blocks per SM so load/store phases
        // of one block hide behind the butterflies of the others; G=2 keeps 64-byte contiguous runs.
        int logG = 1;
        if (!pp.is_last) { if (logG > logB) logG = logB; }
        else if (plan.m > 1) { if (logG > plan.radix_log[0]) logG = plan.radix_log[0]; }
        else logG = 0;
        while (pp.r + logG - 1 > 9) logG--;  // at most 512 threads per block
        pp.logG = logG;
        const int tile = 1 << (pp.r + logG);
        const int threads = tile / 2 > 32 ? tile / 2 : 32;
        const unsigned blocks = (unsigned)(n >> (pp.r + logG));
        const uint4 *src = (t == 0) ? d_data : scratch;
        uint4 *dst = pp.is_last ? d_data : scratch;
        ntt_pass_kernel<P><<<blocks, threads, (size_t)tile * 32, st>>>(src, dst, pp);
        AB_LAUNCHED();
        log_seg = logB;
    }
    if (scratch) AB_CUDA(cudaFreeAsync(scratch, st));

    if (has_coset && inverse) {  // distribute_powers_and_mul_by_const(x, offset_inv, size_inv): 1/n already applied
        uint32_t oinv[8];
        F::inv(oinv, off);
        for (int i = 0; i < 8; i++) g_arg.v[i] = oinv[i];
        size_t threads = (n + 15) / 16;
        distribute_powers_kernel<P><<<(unsigned)((threads + 127) / 128), 128, 0, st>>>(d_data, n, g_arg, one_arg);
        AB_LAUNCHED();
    }
    return 0;
}

int ntt_dispatch(int field, void *d_data, uint32_t log_n, int inverse, const uint64_t *coset, cudaStream_t st) {
    if (!d_data) { set_last_error("null data pointer"); return B200_EINVAL; }
    if (log_n > 40) { set_last_error("log_n out of range"); return B200_ETOOLARGE; }
    switch (field) {
        case B200_FIELD_BLS12_381_FR: return ntt_run<BlsFr>(field, (uint4 *)d_data, (int)log_n, inverse != 0, coset, st);
        case B200_FIELD_BN254_FR: return ntt_run<BnFr>(field, (uint4 *)d_data, (int)log_n, inverse != 0, coset, st);
    }
    set_last_error("unknown scalar field id");
    return B200_EINVAL;
}

}  // namespace ab200
