// point_ntt.cu — radix-2 FFT / inverse FFT whose coefficients are G1 points (Jacobian, Montgomery) and whose domain is the
// curve's scalar field Fr, for sm_90a.
//
// Replaces Radix2EvaluationDomain::{fft_in_place, ifft_in_place} for T = Projective<g1::Config> (T: DomainCoeff<Fr>,
// poly/src/domain/mod.rs:332-361) after the resize step, following fft.rs:74-88 with T = Projective:
//   forward:  [distribute_powers(h)]  io_helper (DIF, butterfly_fn_io :190-198)  derange
//   inverse:  derange  oi_helper (DIT, butterfly_fn_oi :201-210)  distribute_powers_and_mul_by_const(h^-1 or 1, 1/n)
// A point times a field element is `MulAssign<F>` -> mul_bigint over the element's canonical (into_bigint) value; here it is a
// fixed-window signed-digit ladder of complete Jacobian doublings and additions (ec.cuh), so P + P and P - P inside the ladder
// and the butterflies are handled.  Any point with z = 0 is the identity; every identity this unit writes is (R, R, 0).
//
// Launches per call (log_n = k, n = 2^k):
//   forward : (k > 0 ? 1 twiddle table : 0) + (coset ? 1 scale : 0) + k stages + 1 derange
//   inverse : (k > 0 ? 1 twiddle table : 0) + 1 derange + k stages + 1 scale (1/n, or h^-1 and 1/n)
// Work: (n/2)·k butterflies, of which n - 1 have twiddle 1 (no ladder); one ladder per element for each scale pass.
#include "common.cuh"
#include "ec.cuh"
#include "host_api.h"

namespace ab200 {

// Window width of the twiddle ladder.  Signed digits in [-2^(W-1), 2^(W-1)], so the per-thread table holds 1P .. 2^(W-1)P.
// Per ladder on a 255-bit scalar at W = 5: ~250 doublings, ~50 additions and a 16-entry table (1 doubling, 14 additions), ~2.8k
// field multiplications.  W = 5 measured 1.5-3.6 % faster than W = 4 on the H100 at the same register count; its table doubles
// the stack (DESIGN §3.5).
static constexpr int kPointWindow = 5;
static constexpr int kPointHalf = 1 << (kPointWindow - 1);
static constexpr int kPointDigits = (256 + kPointWindow - 1) / kPointWindow;   // k < 2^255: the top window never carries out
static constexpr int kPointThreads = 128;

template <int L> __device__ __forceinline__ void load_point(Jac<L> &p, const uint32_t *src) {
    load_limbs<L>(p.x, src);
    load_limbs<L>(p.y, src + L);
    load_limbs<L>(p.z, src + 2 * L);
}
// identities leave as (R, R, 0) whatever their x and y were
template <class P> __device__ __forceinline__ void store_point(uint32_t *dst, Jac<P::L> &p) {
    using E = Ec<Fp<P>>;
    if (E::jac_is_zero(p)) E::jac_set_zero(p);
    store_limbs<P::L>(dst, p.x);
    store_limbs<P::L>(dst + P::L, p.y);
    store_limbs<P::L>(dst + 2 * P::L, p.z);
}

// p <- k·p for a canonical 256-bit k (8 little-endian words).  Digits are recoded LSB first with d > 2^(W-1) borrowing from the
// next window, then the ladder runs MSB first: W doublings and at most one addition of ±table[|d|-1] per window.
template <class P> __device__ __noinline__ void jac_mul_canonical(Jac<P::L> &p, const uint32_t *k) {
    using E = Ec<Fp<P>>;
    using J = Jac<P::L>;
    int8_t dig[kPointDigits];
    int carry = 0;
#pragma unroll 1
    for (int w = 0; w < kPointDigits; w++) {
        const int bit = w * kPointWindow, word = bit >> 5, sh = bit & 31;
        uint64_t two = k[word];
        if (word + 1 < 8) two |= (uint64_t)k[word + 1] << 32;
        int d = (int)((two >> sh) & ((1u << kPointWindow) - 1)) + carry;
        carry = d > kPointHalf;
        if (carry) d -= 1 << kPointWindow;
        dig[w] = (int8_t)d;
    }
    J tab[kPointHalf];   // dynamically indexed: local memory
    tab[0] = p;
    tab[1] = p;
    E::jac_dbl(tab[1]);
#pragma unroll 1
    for (int m = 2; m < kPointHalf; m++) {
        tab[m] = tab[m - 1];
        E::jac_add(tab[m], p);
    }
    E::jac_set_zero(p);
#pragma unroll 1
    for (int w = kPointDigits - 1; w >= 0; w--) {
#pragma unroll 1
        for (int s = 0; s < kPointWindow; s++) E::jac_dbl(p);
        const int d = dig[w];
        if (d) {
            J t = tab[(d < 0 ? -d : d) - 1];
            if (d < 0) Fp<P>::neg(t.y, t.y);
            E::jac_add(p, t);
        }
    }
}

// tw[k] = canonical limbs of w^k, k < half; 16 consecutive k per thread
template <class PR> __global__ void point_twiddles_kernel(uint4 *tw, size_t half, LimbArg<8> w) {
    using F = Fp<PR>;
    const int CH = 16;
    const size_t k0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * CH;
    if (k0 >= half) return;
    uint32_t cur[8], c[8];
    F::pow_u64(cur, w.v, k0);
    for (size_t k = k0; k < k0 + CH && k < half; k++) {
        F::from_mont(c, cur);
        tw[2 * k] = make_uint4(c[0], c[1], c[2], c[3]);
        tw[2 * k + 1] = make_uint4(c[4], c[5], c[6], c[7]);
        F::mul(cur, cur, w.v);
    }
}

// One radix-2 stage with half-distance `gap` = 2^log_gap over n = 2^log_n points; one butterfly per thread.  Threads are
// twiddle-major: t = j * chunks + chunk, so with >= 32 chunks a warp shares j and its twiddle (uniform digit loops).
//   DIF (forward, fft.rs:190-198): lo' = lo + hi, hi' = (lo - hi)·w^j
//   DIT (inverse, fft.rs:201-210): hi *= w^j, lo' = lo + hi, hi' = lo - hi
// with w^j = tw[j * chunks] (the table holds w^k, k < n/2, w the n-th root of this direction).
template <class PQ, bool DIT> __global__ void __launch_bounds__(kPointThreads) point_ntt_stage_kernel(uint32_t *pts, const uint4 *tw, int log_n, int log_gap) {
    using E = Ec<Fp<PQ>>;
    constexpr int L = PQ::L;
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= ((size_t)1 << (log_n - 1))) return;
    const int log_chunks = log_n - 1 - log_gap;
    const size_t j = t >> log_chunks, chunk = t & (((size_t)1 << log_chunks) - 1);
    const size_t lo = (chunk << (log_gap + 1)) + j, hi = lo + ((size_t)1 << log_gap);
    uint32_t *plo = pts + lo * 3 * L, *phi = pts + hi * 3 * L;
    Jac<L> a, b;
    load_point<L>(a, plo);
    load_point<L>(b, phi);
    uint32_t k[8];
    if (j) {
        const uint4 *tp = tw + 2 * (j << log_chunks);
        const uint4 k0 = __ldg(tp), k1 = __ldg(tp + 1);
        k[0] = k0.x; k[1] = k0.y; k[2] = k0.z; k[3] = k0.w; k[4] = k1.x; k[5] = k1.y; k[6] = k1.z; k[7] = k1.w;
    }
    if (DIT && j) jac_mul_canonical<PQ>(b, k);
    Jac<L> d = b;
    Fp<PQ>::neg(d.y, d.y);
    E::jac_add(d, a);       // lo - hi
    E::jac_add(a, b);       // lo + hi
    if (!DIT && j) jac_mul_canonical<PQ>(d, k);
    store_point<PQ>(plo, a);
    store_point<PQ>(phi, d);
}

// x[i] *= c·g^i  (distribute_powers_and_mul_by_const, poly/src/domain/mod.rs:119-148); one point per thread
template <class PQ, class PR> __global__ void __launch_bounds__(kPointThreads) point_scale_kernel(uint32_t *pts, size_t n, LimbArg<8> g, LimbArg<8> c) {
    using FR = Fp<PR>;
    constexpr int L = PQ::L;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t s[8], k[8];
    FR::pow_u64(s, g.v, i);
    FR::mul(s, s, c.v);
    FR::from_mont(k, s);
    Jac<L> p;
    load_point<L>(p, pts + i * 3 * L);
    jac_mul_canonical<PQ>(p, k);
    store_point<PQ>(pts + i * 3 * L, p);
}

// derange (fft.rs:373-380): swap i and bitrev(i) for i < bitrev(i), in place; every element is written once, identities canonical
template <class PQ> __global__ void point_derange_kernel(uint32_t *pts, int log_n) {
    constexpr int L = PQ::L;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ((size_t)1 << log_n)) return;
    const size_t r = log_n ? (size_t)(__brevll((unsigned long long)i) >> (64 - log_n)) : 0;
    if (i > r) return;
    Jac<L> a, b;
    load_point<L>(a, pts + i * 3 * L);
    if (i == r) { store_point<PQ>(pts + i * 3 * L, a); return; }
    load_point<L>(b, pts + r * 3 * L);
    store_point<PQ>(pts + i * 3 * L, b);
    store_point<PQ>(pts + r * 3 * L, a);
}

template <class PR> static void point_root_of_unity(uint32_t *g, int log_n) {   // get_root_of_unity, ff/src/fields/fft_friendly.rs:66-82
    for (int i = 0; i < 8; i++) g[i] = PR::TWO_ADIC_ROOT(i);
    for (int i = log_n; i < PR::TWO_ADICITY; i++) Fp<PR>::sqr(g, g);
}

static unsigned point_blocks(size_t threads) { return (unsigned)((threads + kPointThreads - 1) / kPointThreads); }

template <class PQ, class PR> static int point_ntt_run(uint32_t *d, int log_n, bool inverse, const uint64_t *coset, cudaStream_t st) {
    using FR = Fp<PR>;
    if (log_n > PR::TWO_ADICITY) {
        set_last_error("log_n exceeds TWO_ADICITY (Radix2EvaluationDomain::new would return None)");
        return B200_ETOOLARGE;
    }
    const size_t n = (size_t)1 << log_n;
    LimbArg<8> one, h, w, size_inv;
    FR::set_one(one.v);
    bool has_coset = false;
    if (coset) {
        for (int i = 0; i < 4; i++) {
            h.v[2 * i] = (uint32_t)coset[i];
            h.v[2 * i + 1] = (uint32_t)(coset[i] >> 32);
        }
        has_coset = !limbs_eq<8>(h.v, one.v);   // `if !self.offset.is_one()` fft.rs:75
    }
    point_root_of_unity<PR>(w.v, log_n);
    if (inverse) FR::inv(w.v, w.v);
    uint4 *tw = nullptr;
    if (log_n > 0) {
        AB_CUDA(cudaMallocAsync(&tw, (n / 2) * 32, st));
        point_twiddles_kernel<PR><<<(unsigned)((n / 2 + 16 * 128 - 1) / (16 * 128)), 128, 0, st>>>(tw, n / 2, w);
        AB_LAUNCHED();
    }
    const size_t half = n / 2;
    if (!inverse) {
        if (has_coset) {
            point_scale_kernel<PQ, PR><<<point_blocks(n), kPointThreads, 0, st>>>(d, n, h, one);
            AB_LAUNCHED();
        }
        for (int lg = log_n - 1; lg >= 0; lg--) {
            point_ntt_stage_kernel<PQ, false><<<point_blocks(half), kPointThreads, 0, st>>>(d, tw, log_n, lg);
            AB_LAUNCHED();
        }
        point_derange_kernel<PQ><<<point_blocks(n), kPointThreads, 0, st>>>(d, log_n);
        AB_LAUNCHED();
    } else {
        point_derange_kernel<PQ><<<point_blocks(n), kPointThreads, 0, st>>>(d, log_n);
        AB_LAUNCHED();
        for (int lg = 0; lg < log_n; lg++) {
            point_ntt_stage_kernel<PQ, true><<<point_blocks(half), kPointThreads, 0, st>>>(d, tw, log_n, lg);
            AB_LAUNCHED();
        }
        uint32_t nn[8] = {(uint32_t)n, (uint32_t)((uint64_t)n >> 32), 0, 0, 0, 0, 0, 0};   // size_inv (radix2/mod.rs:74)
        FR::to_mont(nn, nn);
        FR::inv(size_inv.v, nn);
        LimbArg<8> g = one;
        if (has_coset) FR::inv(g.v, h.v);
        point_scale_kernel<PQ, PR><<<point_blocks(n), kPointThreads, 0, st>>>(d, n, g, size_inv);
        AB_LAUNCHED();
    }
    if (tw) AB_CUDA(cudaFreeAsync(tw, st));
    return 0;
}

int point_ntt_check(int curve, const void *points, uint32_t log_n) {
    if (curve != B200_CURVE_BLS12_381 && curve != B200_CURVE_BN254) {
        set_last_error(curve == B200_CURVE_BLS12_381_G2 ? "G2 points are not supported by the point FFT" : "unknown curve id");
        return B200_EINVAL;
    }
    if (!points) { set_last_error("null points pointer"); return B200_EINVAL; }
    if (log_n > (uint32_t)field_info(curve_info(curve)->scalar_field)->two_adicity) {
        set_last_error("log_n exceeds TWO_ADICITY (Radix2EvaluationDomain::new would return None)");
        return B200_ETOOLARGE;
    }
    return 0;
}

int point_ntt_dispatch(int curve, void *d_points, uint32_t log_n, int inverse, const uint64_t *coset, cudaStream_t st) {
    if (int rc = point_ntt_check(curve, d_points, log_n)) return rc;
    if (curve == B200_CURVE_BLS12_381) return point_ntt_run<BlsFq, BlsFr>((uint32_t *)d_points, (int)log_n, inverse != 0, coset, st);
    return point_ntt_run<BnFq, BnFr>((uint32_t *)d_points, (int)log_n, inverse != 0, coset, st);
}

}  // namespace ab200
