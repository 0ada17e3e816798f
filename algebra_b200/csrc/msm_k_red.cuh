// msm_k_red.cuh — bucket reduction, window combine, Jacobian sum / normalisation kernels and their launchers.
#pragma once
#include "msm_common.cuh"

namespace ab200 {

// ------------------------------------------------------------------------------------------------
// bucket reduction.  Window w needs S_w = sum_j (j+1) * B_w[j]  (:478-484).  Thread t of a window takes buckets
// [t*m, (t+1)*m): running sum gives  sum_l (l+1)*B[t*m+l]  and the chunk total R_t; adding (t*m) * R_t (double-and-add)
// makes its contribution complete (for a bucket slice starting at bucket `off` of the window: (off + t*m) * R_t).
// partial index = window * chunks_stride + t.
// ------------------------------------------------------------------------------------------------
template <class C>
__global__ void __launch_bounds__(128) msm_bucket_reduce_kernel(const uint32_t *__restrict__ buckets, MsmGeom g, int log_m,
                                                                uint32_t chunks_per_window, uint32_t *__restrict__ partials) {
    using F = typename C::F;
    using E = Ec<F>;
    constexpr int L = F::L;
    uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t w = tid / chunks_per_window, t = tid % chunks_per_window;
    if (w >= (uint32_t)g.W) return;
    const uint32_t nbw = (w == (uint32_t)g.W - 1) ? g.nb_top : g.nb;
    const uint32_t m = 1u << log_m;
    typename E::B run, sum;
    E::xyzz_set_zero(run);
    E::xyzz_set_zero(sum);
    const uint32_t lo = t * m;
    if (lo < nbw) {
        const uint32_t hi = min(lo + m, nbw);
        const uint32_t *base = buckets + ((size_t)w * g.nb) * (4 * L);
        for (uint32_t j = hi; j-- > lo;) {
            typename E::B b;
            load_xyzz<L>(b, base + (size_t)j * (4 * L));
            E::xyzz_add(run, b);
            E::xyzz_add(sum, run);
        }
        // sum += (lo + first bucket of the slice) * run
        const uint32_t wlo = lo + ((w == (uint32_t)g.W - 1) ? g.off_top : g.off);
        if (wlo != 0 && !E::xyzz_is_zero(run)) {
            typename E::B acc;
            E::xyzz_set_zero(acc);
            for (int bit = 31 - __clz(wlo); bit >= 0; bit--) {
                if (!E::xyzz_is_zero(acc)) E::xyzz_dbl(acc);
                if ((wlo >> bit) & 1) E::xyzz_add(acc, run);
            }
            E::xyzz_add(sum, acc);
        }
    }
    store_xyzz<L>(partials + ((size_t)w * chunks_per_window + t) * (4 * L), sum);
}

// Block (w, s) of a window sums `per_block` consecutive partials of window w (strided over the threads, then a shared-memory
// tree) -> out[w * blocks_per_window + s].  Run twice (chunks -> 32 per window -> 1): the additions are latency-bound
// (~14 dependent multiplications each), so the depth per thread — not the count — is what costs.
template <class C>
__global__ void __launch_bounds__(128) msm_sum_partials_kernel(const uint32_t *__restrict__ partials, uint32_t chunks_per_window, uint32_t per_block,
                                                               uint32_t blocks_per_window, uint32_t *__restrict__ window_sums) {
    using F = typename C::F;
    using E = Ec<F>;
    constexpr int L = F::L;
    extern __shared__ uint32_t sm[];
    const uint32_t w = blockIdx.x / blocks_per_window, sblk = blockIdx.x % blocks_per_window;
    const uint32_t t_lo = sblk * per_block, t_hi = min(chunks_per_window, t_lo + per_block);
    typename E::B acc;
    E::xyzz_set_zero(acc);
    for (uint32_t t = t_lo + threadIdx.x; t < t_hi; t += blockDim.x) {
        typename E::B b;
        load_xyzz<L>(b, partials + ((size_t)w * chunks_per_window + t) * (4 * L));
        E::xyzz_add(acc, b);
    }
    store_xyzz<L>(sm + threadIdx.x * (4 * L), acc);
    __syncthreads();
    for (uint32_t s = blockDim.x >> 1; s > 0; s >>= 1) {
        if (threadIdx.x < s) {
            typename E::B a, b;
            load_xyzz<L>(a, sm + threadIdx.x * (4 * L));
            load_xyzz<L>(b, sm + (threadIdx.x + s) * (4 * L));
            E::xyzz_add(a, b);
            store_xyzz<L>(sm + threadIdx.x * (4 * L), a);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        typename E::B a;
        load_xyzz<L>(a, sm);
        store_xyzz<L>(window_sums + (size_t)blockIdx.x * (4 * L), a);
    }
}

// Window combine: total = sum_w 2^(c*w) * S_w by Horner (:489-502), Projective += &Bucket (bucket.rs:345-359); Jacobian result
// (x, y, z) -> out (3L words).  The independent field multiplications of every point operation are spread over the lanes of one
// warp (operands in shared-memory slots): a Jacobian doubling is 3 dependent rounds of multiplications instead of 7, an
// addition 6 instead of 16.  c*(W-1) doublings in sequence are the latency floor of this step, a
// large share of a small MSM; the exceptional cases (equal / opposite operands)
// fall back to the one-thread formulas (Ec::jac_add).
template <class F> struct CoopSlots {
    static constexpr int L = F::L;
    uint32_t *sm;
    __device__ __forceinline__ uint32_t *at(int slot) const { return sm + slot * L; }
    // dst[i] = a[i] * b[i] for i < n, lane i does product i
    __device__ __forceinline__ void mul(int n, int d0, int a0, int b0, int d1 = 0, int a1 = 0, int b1 = 0, int d2 = 0, int a2 = 0, int b2 = 0, int d3 = 0,
                                        int a3 = 0, int b3 = 0) const {
        const int lane = threadIdx.x & 31;
        __syncwarp();   // every lane has finished reading the slots (uniform branch conditions) before any of them is overwritten
        if (lane < n) {
            const int d = lane == 0 ? d0 : lane == 1 ? d1 : lane == 2 ? d2 : d3;
            const int a = lane == 0 ? a0 : lane == 1 ? a1 : lane == 2 ? a2 : a3;
            const int b = lane == 0 ? b0 : lane == 1 ? b1 : lane == 2 ? b2 : b3;
            uint32_t x[L], y[L];
#pragma unroll
            for (int i = 0; i < L; i++) { x[i] = at(a)[i]; y[i] = at(b)[i]; }
            F::mul(x, x, y);
#pragma unroll
            for (int i = 0; i < L; i++) at(d)[i] = x[i];
        }
        __syncwarp();
    }
};

template <class C> __global__ void __launch_bounds__(32) msm_window_combine_coop_kernel(const uint32_t *__restrict__ window_sums, int W, int c,
                                                                                       uint32_t *__restrict__ out) {
    using F = typename C::F;
    using E = Ec<F>;
    constexpr int L = F::L;
    enum { X = 0, Y, Z, X2, Y2, Z2, T0, T1, T2, T3, T4, T5, T6, T7, NSLOT };
    __shared__ uint32_t sm[NSLOT * L];
    CoopSlots<F> S{sm};
    const int lane = threadIdx.x;
    // (the leading __syncwarp keeps lane 0 from overwriting a slot that another lane is still reading for a warp-uniform test:
    // lanes of a warp are not guaranteed to run in lockstep — compute-sanitizer racecheck flagged exactly that)
    auto lane0 = [&](auto fn) { __syncwarp(); if (lane == 0) fn(); __syncwarp(); };
    lane0([&] { F::set_one(S.at(X)); F::set_one(S.at(Y)); F::set_zero(S.at(Z)); });
    for (int w = W - 1; w >= 0; w--) {
        // ---- operand: XYZZ window sum -> Jacobian (x*zz, y*zzz, zz)  (From<Bucket> for Projective, bucket.rs:389-398)
        lane0([&] {
            const uint32_t *p = window_sums + (size_t)w * (4 * L);
#pragma unroll
            for (int i = 0; i < L; i++) { S.at(X2)[i] = p[i]; S.at(Y2)[i] = p[L + i]; S.at(Z2)[i] = p[2 * L + i]; S.at(T0)[i] = p[3 * L + i]; }
        });
        const bool op_zero = limbs_is_zero<L>(S.at(Z2)) && limbs_is_zero<L>(S.at(T0));
        if (!op_zero) {
            S.mul(2, X2, X2, Z2, Y2, Y2, T0);
            if (limbs_is_zero<L>(S.at(Z))) {   // total is the identity: total = operand
                lane0([&] { limbs_copy<L>(S.at(X), S.at(X2)); limbs_copy<L>(S.at(Y), S.at(Y2)); limbs_copy<L>(S.at(Z), S.at(Z2)); });
            } else {   // add-2007-bl (group.rs:450-538), multiplications of equal depth side by side
                S.mul(2, T0, Z, Z, T1, Z2, Z2);                                   // z1z1, z2z2
                S.mul(4, T2, X, T1, T3, X2, T0, T4, Y, Z2, T5, Y2, Z);            // u1, u2, y1*z2, y2*z1
                S.mul(3, T4, T4, T1, T5, T5, T0, T6, Z, Z2);                      // s1, s2, z1*z2
                const bool same_x = limbs_eq<L>(S.at(T2), S.at(T3));
                if (same_x) {   // doubling or cancellation: the one-thread formulas handle it
                    lane0([&] {
                        typename E::J a, b;
                        limbs_copy<L>(a.x, S.at(X)); limbs_copy<L>(a.y, S.at(Y)); limbs_copy<L>(a.z, S.at(Z));
                        limbs_copy<L>(b.x, S.at(X2)); limbs_copy<L>(b.y, S.at(Y2)); limbs_copy<L>(b.z, S.at(Z2));
                        E::jac_add(a, b);
                        limbs_copy<L>(S.at(X), a.x); limbs_copy<L>(S.at(Y), a.y); limbs_copy<L>(S.at(Z), a.z);
                    });
                } else {
                    lane0([&] {
                        F::sub(S.at(T0), S.at(T3), S.at(T2));          // h = u2 - u1
                        F::dbl(S.at(T1), S.at(T0));                    // 2h
                        F::sub(S.at(T3), S.at(T5), S.at(T4));          // s2 - s1
                        F::dbl(S.at(T3), S.at(T3));                    // r
                        F::dbl(S.at(T4), S.at(T4));                    // 2 s1
                    });
                    S.mul(1, T1, T1, T1);                                             // i = (2h)^2
                    S.mul(3, T5, T0, T1, T2, T2, T1, T7, T3, T3);                     // h*i, v = u1*i, r^2
                    lane0([&] {
                        F::sub(S.at(X), S.at(T7), S.at(T5));           // x3 = r^2 - h i - 2 v
                        F::dbl(S.at(T7), S.at(T2));
                        F::sub(S.at(X), S.at(X), S.at(T7));
                        F::sub(S.at(T2), S.at(T2), S.at(X));           // v - x3
                    });
                    S.mul(3, T2, T3, T2, T4, T4, T5, T6, T6, T0);                     // r (v - x3), 2 s1 h i, z1 z2 h
                    lane0([&] {
                        F::sub(S.at(Y), S.at(T2), S.at(T4));
                        F::dbl(S.at(Z), S.at(T6));
                    });
                }
            }
        }
        if (w > 0 && !limbs_is_zero<L>(S.at(Z))) {
            for (int d = 0; d < c; d++) {   // dbl-2009-l as in Ec::jac_dbl (group.rs:171-221)
                S.mul(3, T0, X, X, T1, Y, Y, T2, Z, Y);                               // a, b, z*y
                lane0([&] {
                    F::dbl(S.at(Z), S.at(T2));                         // z3 = 2 z y
                    F::dbl(S.at(T3), S.at(T0));
                    F::add(S.at(T3), S.at(T3), S.at(T0));              // e = 3 a
                });
                S.mul(3, T4, T1, T1, T5, X, T1, T6, T3, T3);                          // c = b^2, x*b, e^2
                lane0([&] {
                    F::dbl(S.at(T5), S.at(T5));
                    F::dbl(S.at(T5), S.at(T5));                        // d = 4 x b
                    F::dbl(S.at(T7), S.at(T5));
                    F::sub(S.at(X), S.at(T6), S.at(T7));               // x3 = e^2 - 2 d
                    F::sub(S.at(T5), S.at(T5), S.at(X));               // d - x3
                    F::dbl(S.at(T4), S.at(T4));
                    F::dbl(S.at(T4), S.at(T4));
                    F::dbl(S.at(T4), S.at(T4));                        // 8 c
                });
                S.mul(1, T5, T5, T3);
                lane0([&] { F::sub(S.at(Y), S.at(T5), S.at(T4)); });
            }
        }
    }
    if (lane == 0) {
        if (limbs_is_zero<L>(S.at(Z))) { F::set_one(S.at(X)); F::set_one(S.at(Y)); }   // Projective::zero() = (1, 1, 0)
        store_limbs<L>(out, S.at(X));
        store_limbs<L>(out + L, S.at(Y));
        store_limbs<L>(out + 2 * L, S.at(Z));
    }
}

// sum of k Jacobian points (multi-GPU gather reduce), one thread
template <class C> __global__ void jac_sum_kernel(const uint32_t *__restrict__ pts, size_t k, uint32_t *__restrict__ out) {
    using F = typename C::F;
    using E = Ec<F>;
    constexpr int L = F::L;
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    typename E::J total;
    E::jac_set_zero(total);
    for (size_t i = 0; i < k; i++) {
        typename E::J j;
        load_limbs<L>(j.x, pts + i * 3 * L);
        load_limbs<L>(j.y, pts + i * 3 * L + L);
        load_limbs<L>(j.z, pts + i * 3 * L + 2 * L);
        E::jac_add(total, j);
    }
    if (E::jac_is_zero(total)) E::jac_set_zero(total);
    store_limbs<L>(out, total.x);
    store_limbs<L>(out + L, total.y);
    store_limbs<L>(out + 2 * L, total.z);
}
template <class C> __global__ void jac_to_affine_kernel(const uint32_t *__restrict__ pts, size_t k, uint32_t *__restrict__ out) {
    using F = typename C::F;
    using E = Ec<F>;
    constexpr int L = F::L;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= k) return;
    typename E::J j;
    load_limbs<L>(j.x, pts + i * 3 * L);
    load_limbs<L>(j.y, pts + i * 3 * L + L);
    load_limbs<L>(j.z, pts + i * 3 * L + 2 * L);
    uint32_t ax[L], ay[L];
    E::jac_to_affine(ax, ay, j);
    store_limbs<L>(out + i * 2 * L, ax);
    store_limbs<L>(out + i * 2 * L + L, ay);
}

template <class C>
int MsmRedLaunch<C>::reduce(const uint32_t *buckets, MsmGeom g, int log_m, uint32_t chunks, uint32_t *partials, uint32_t *partials2, uint32_t *window_sums,
                            cudaStream_t st) {
    constexpr int L = C::F::L;
    const unsigned rthreads = (unsigned)g.W * chunks;
    msm_bucket_reduce_kernel<C><<<(rthreads + 127) / 128, 128, 0, st>>>(buckets, g, log_m, chunks, partials);
    AB_LAUNCHED();
    AB_CUDA(cudaFuncSetAttribute(msm_sum_partials_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 4 * L * 4));
    if (chunks > 1024) {   // two rounds: chunks -> S per window (in place at the front of `partials`' second half is not needed: `stage2`), S -> 1
        const uint32_t S = 32, per = (chunks + S - 1) / S;
        uint32_t *stage2 = partials2;
        msm_sum_partials_kernel<C><<<g.W * S, 128, 128 * 4 * L * 4, st>>>(partials, chunks, per, S, stage2);
        AB_LAUNCHED();
        msm_sum_partials_kernel<C><<<g.W, 128, 128 * 4 * L * 4, st>>>(stage2, S, S, 1, window_sums);
    } else {
        msm_sum_partials_kernel<C><<<g.W, 128, 128 * 4 * L * 4, st>>>(partials, chunks, chunks, 1, window_sums);
    }
    AB_LAUNCHED();
    return 0;
}
template <class C> int MsmRedLaunch<C>::combine(const uint32_t *window_sums, int W, int c, uint32_t *out, cudaStream_t st) {
    msm_window_combine_coop_kernel<C><<<1, 32, 0, st>>>(window_sums, W, c, out);
    AB_LAUNCHED();
    return 0;
}
template <class C> int MsmRedLaunch<C>::sum_or_affine(bool to_affine, const uint32_t *d_in, size_t k, uint32_t *d_out, cudaStream_t st) {
    if (to_affine) jac_to_affine_kernel<C><<<(unsigned)((k + 31) / 32), 32, 0, st>>>(d_in, k, d_out);
    else jac_sum_kernel<C><<<1, 32, 0, st>>>(d_in, k, d_out);
    AB_LAUNCHED();
    return 0;
}

}  // namespace ab200
