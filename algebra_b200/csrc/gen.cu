// gen.cu — synthetic inputs generated on the device (benchmarks, large-size property tests).
//   scalars: uniform Fr by mask-and-reject, the rule of Fp::rand (ff/src/fields/models/fp/mod.rs:521-548)
//   bases:   P_i = b_i * G (b_i a 64-bit splitmix64 stream), fixed-base comb over an 8 x 256 table of multiples of G,
//            normalised to affine with a per-thread batch inversion (the role of Projective::normalize_batch,
//            group.rs:302-319) — so that the exact MSM answer is (sum s_i * b_i mod r) * G.
#include <map>
#include <mutex>

#include "common.cuh"
#include "host_api.h"
#include "ec.cuh"

namespace ab200 {

static constexpr int kGenBatch = 8;  // points normalised with one inversion per thread

__host__ __device__ __forceinline__ uint64_t splitmix64_at(uint64_t seed, uint64_t idx) {
    uint64_t z = seed + (idx + 1) * 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

template <class P> __global__ void gen_scalars_kernel(uint64_t seed, size_t n, uint32_t *out) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t v[8];
    for (uint64_t attempt = 0;; attempt++) {
#pragma unroll
        for (int k = 0; k < 4; k++) {
            uint64_t w = splitmix64_at(seed ^ (attempt * 0xD1B54A32D192ED03ull), i * 4 + k);
            v[2 * k] = (uint32_t)w;
            v[2 * k + 1] = (uint32_t)(w >> 32);
        }
        v[7] &= (P::BITS % 32) ? ((1u << (P::BITS % 32)) - 1) : 0xffffffffu;
        // accept iff v < p
        uint32_t t = ptx::sub_cc(v[0], P::MOD(0));
#pragma unroll
        for (int k = 1; k < 8; k++) t = ptx::subc_cc(v[k], P::MOD(k));
        (void)t;
        if (ptx::subc(0u, 0u)) break;
    }
    store_limbs<8>(out + i * 8, v);
}

// generator traits: coordinate-field operations class + the generator's affine coordinates (Montgomery words)
template <class P> struct GenG1 {
    using F = Fp<P>;
    static __device__ __forceinline__ void generator(uint32_t *x, uint32_t *y) {
#pragma unroll
        for (int i = 0; i < P::L; i++) { x[i] = P::GEN_X(i); y[i] = P::GEN_Y(i); }
    }
};
struct GenBlsG2 {
    using F = Fp2<BlsFq>;
    static __device__ __forceinline__ void generator(uint32_t *x, uint32_t *y) {
#pragma unroll
        for (int i = 0; i < 24; i++) { x[i] = BlsG2Gen::GEN_X(i); y[i] = BlsG2Gen::GEN_Y(i); }
    }
};

// table[w*256 + d] = (d * 256^w) * G, affine Montgomery (d = 0 -> (0,0))
template <class G> __global__ void gen_table_kernel(uint32_t *table) {
    using F = typename G::F;
    using E = Ec<F>;
    constexpr int L = F::L;
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 8 * 256) return;
    int w = t >> 8, d = t & 255;
    typename E::J base, acc;
    G::generator(base.x, base.y);
    F::set_one(base.z);
#pragma unroll 1
    for (int k = 0; k < 8 * w; k++) E::jac_dbl(base);
    E::jac_set_zero(acc);
#pragma unroll 1
    for (int bit = 7; bit >= 0; bit--) {
        E::jac_dbl(acc);
        if ((d >> bit) & 1) E::jac_add(acc, base);
    }
    uint32_t ax[L], ay[L];
    E::jac_to_affine(ax, ay, acc);
    store_limbs<L>(table + (size_t)t * 2 * L, ax);
    store_limbs<L>(table + (size_t)t * 2 * L + L, ay);
}

template <class G> __global__ void __launch_bounds__(64) gen_bases_kernel(uint64_t seed, size_t n, const uint32_t *__restrict__ table,
                                                                         uint32_t *__restrict__ bases, uint64_t *__restrict__ bvals) {
    using F = typename G::F;
    using E = Ec<F>;
    constexpr int L = F::L;
    size_t i0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * kGenBatch;
    if (i0 >= n) return;
    typename E::B pts[kGenBatch];
    uint32_t prefix[kGenBatch][L];
    int cnt = 0;
#pragma unroll 1
    for (; cnt < kGenBatch && i0 + cnt < n; cnt++) {
        uint64_t b = splitmix64_at(seed, i0 + cnt) | 1ull;
        if (bvals) bvals[i0 + cnt] = b;
        typename E::B acc;
        E::xyzz_set_zero(acc);
#pragma unroll 1
        for (int w = 0; w < 8; w++) {
            uint32_t d = (uint32_t)(b >> (8 * w)) & 255u;
            uint32_t px[L], py[L];
            const uint32_t *tp = table + (size_t)(w * 256 + d) * 2 * L;
            load_limbs_nc<L>(px, tp);
            load_limbs_nc<L>(py, tp + L);
            E::madd(acc, px, py, false);
        }
        pts[cnt] = acc;
        if (cnt == 0) limbs_copy<L>(prefix[0], acc.zzz);
        else F::mul(prefix[cnt], prefix[cnt - 1], acc.zzz);
    }
    // b*G with b odd and < 2^64 << r is never the identity, so every zzz is invertible
    uint32_t inv[L];
    F::inv(inv, prefix[cnt - 1]);
#pragma unroll 1
    for (int k = cnt - 1; k >= 0; k--) {
        uint32_t zi[L], t[L], ax[L], ay[L];
        if (k > 0) F::mul(zi, inv, prefix[k - 1]);
        else limbs_copy<L>(zi, inv);            // zi = 1/zzz_k
        F::mul(inv, inv, pts[k].zzz);
        F::mul(t, pts[k].zz, zi);               // zz/zzz = 1/z ; (1/z)^2 = 1/zz
        F::sqr(t, t);
        F::mul(ax, pts[k].x, t);
        F::mul(ay, pts[k].y, zi);
        store_limbs<L>(bases + (i0 + k) * 2 * L, ax);
        store_limbs<L>(bases + (i0 + k) * 2 * L + L, ay);
    }
}

// ---- fixed-base batch multiplication and batch normalisation as public operations (SURVEY.md §8f rank 2) ----------------
// table[w*256 + d] = (d * 256^w) * B for an arbitrary affine base B, w < windows  (BatchMulPreprocessing::new,
// ec/src/scalar_mul/mod.rs:163-215, with an 8-bit window)
template <class P> __global__ void batch_table_kernel(LimbArg<P::L> bx, LimbArg<P::L> by, int windows, uint32_t *table) {
    using E = Ec<Fp<P>>;
    constexpr int L = P::L;
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= windows * 256) return;
    int w = t >> 8, d = t & 255;
    typename E::J base, acc;
    E::jac_set_zero(base);
    if (!E::affine_is_zero(bx.v, by.v)) {
#pragma unroll
        for (int i = 0; i < L; i++) { base.x[i] = bx.v[i]; base.y[i] = by.v[i]; base.z[i] = P::ONE(i); }
    }
#pragma unroll 1
    for (int k = 0; k < 8 * w; k++) E::jac_dbl(base);
    E::jac_set_zero(acc);
#pragma unroll 1
    for (int bit = 7; bit >= 0; bit--) {
        E::jac_dbl(acc);
        if ((d >> bit) & 1) E::jac_add(acc, base);
    }
    uint32_t ax[L], ay[L];
    E::jac_to_affine(ax, ay, acc);
    store_limbs<L>(table + (size_t)t * 2 * L, ax);
    store_limbs<L>(table + (size_t)t * 2 * L + L, ay);
}

// XYZZ points of one thread -> affine with ONE inversion (Montgomery's trick, ff/src/fields/mod.rs:358-420); identity -> (0,0)
template <class P, int B> __device__ __forceinline__ void xyzz_batch_to_affine(Xyzz<P::L> *pts, int cnt, uint32_t *out /* cnt x 2L */) {
    using E = Ec<Fp<P>>;
    using F = Fp<P>;
    constexpr int L = P::L;
    uint32_t prefix[B][L], run[L];
    F::set_one(run);
#pragma unroll 1
    for (int k = 0; k < cnt; k++) {
        limbs_copy<L>(prefix[k], run);                        // product of the non-identity zzz before k
        if (!E::xyzz_is_zero(pts[k])) F::mul(run, run, pts[k].zzz);
    }
    uint32_t inv[L];
    F::inv(inv, run);
#pragma unroll 1
    for (int k = cnt - 1; k >= 0; k--) {
        uint32_t ax[L], ay[L];
        if (E::xyzz_is_zero(pts[k])) {
            F::set_zero(ax);
            F::set_zero(ay);
        } else {
            uint32_t zi[L], t[L];
            F::mul(zi, inv, prefix[k]);                        // 1/zzz_k
            F::mul(inv, inv, pts[k].zzz);
            F::mul(t, pts[k].zz, zi);                          // zz/zzz = 1/z ; (1/z)^2 = 1/zz
            F::sqr(t, t);
            F::mul(ax, pts[k].x, t);
            F::mul(ay, pts[k].y, zi);
        }
        store_limbs<L>(out + (size_t)k * 2 * L, ax);
        store_limbs<L>(out + (size_t)k * 2 * L + L, ay);
    }
}

// out[i] = scalars[i] * B  (BatchMulPreprocessing::batch_mul, ec/src/scalar_mul/mod.rs:225-245): 32 table additions per scalar
template <class PQ, class PR> __global__ void __launch_bounds__(64) batch_mul_kernel(const uint32_t *__restrict__ scalars, size_t n,
                                                                                    const uint32_t *__restrict__ table, int windows,
                                                                                    uint32_t *__restrict__ out) {
    using E = Ec<Fp<PQ>>;
    using FR = Fp<PR>;
    constexpr int L = PQ::L;
    size_t i0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * kGenBatch;
    if (i0 >= n) return;
    typename E::B pts[kGenBatch];
    int cnt = 0;
#pragma unroll 1
    for (; cnt < kGenBatch && i0 + cnt < n; cnt++) {
        uint32_t s[8], k[8];
        load_limbs_nc<8>(s, scalars + (i0 + cnt) * 8);
        FR::from_mont(k, s);
        typename E::B acc;
        E::xyzz_set_zero(acc);
#pragma unroll 1
        for (int w = 0; w < windows; w++) {
            uint32_t d = (k[w >> 2] >> (8 * (w & 3))) & 255u;
            if (d == 0) continue;
            uint32_t px[L], py[L];
            const uint32_t *tp = table + (size_t)(w * 256 + d) * 2 * L;
            load_limbs_nc<L>(px, tp);
            load_limbs_nc<L>(py, tp + L);
            E::madd(acc, px, py, false);
        }
        pts[cnt] = acc;
    }
    xyzz_batch_to_affine<PQ, kGenBatch>(pts, cnt, out + i0 * 2 * L);
}

// Projective::normalize_batch (group.rs:302-319): Jacobian (x,y,z) -> affine, z = 0 -> identity (0,0)
template <class P> __global__ void __launch_bounds__(64) normalize_batch_kernel(const uint32_t *__restrict__ jac, size_t n, uint32_t *__restrict__ out) {
    using F = Fp<P>;
    constexpr int L = P::L;
    size_t i0 = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * kGenBatch;
    if (i0 >= n) return;
    Xyzz<P::L> pts[kGenBatch];
    int cnt = 0;
#pragma unroll 1
    for (; cnt < kGenBatch && i0 + cnt < n; cnt++) {
        const uint32_t *p = jac + (i0 + cnt) * 3 * L;
        uint32_t z[L];
        load_limbs<L>(pts[cnt].x, p);
        load_limbs<L>(pts[cnt].y, p + L);
        load_limbs<L>(z, p + 2 * L);
        F::sqr(pts[cnt].zz, z);                                // Jacobian z  ->  XYZZ (zz, zzz) = (z^2, z^3)
        F::mul(pts[cnt].zzz, pts[cnt].zz, z);
    }
    xyzz_batch_to_affine<P, kGenBatch>(pts, cnt, out + i0 * 2 * L);
}

static std::mutex g_table_mutex;
static std::map<std::pair<int, int>, uint32_t *> g_tables;

template <class G> static int gen_bases_run(int curve, uint64_t seed, size_t n, void *d_bases, void *d_b, cudaStream_t st) {
    constexpr int L = G::F::L;
    int dev = 0;
    AB_CUDA(cudaGetDevice(&dev));
    uint32_t *table = nullptr;
    {
        std::lock_guard<std::mutex> lk(g_table_mutex);
        auto key = std::make_pair(dev, curve);
        auto it = g_tables.find(key);
        if (it == g_tables.end()) {
            AB_CUDA(cudaMalloc(&table, (size_t)8 * 256 * 2 * L * 4));
            gen_table_kernel<G><<<(8 * 256 + 63) / 64, 64, 0, st>>>(table);
            AB_LAUNCHED();
            AB_CUDA(cudaStreamSynchronize(st));
            g_tables[key] = table;
        } else table = it->second;
    }
    size_t threads = (n + kGenBatch - 1) / kGenBatch;
    gen_bases_kernel<G><<<(unsigned)((threads + 63) / 64), 64, 0, st>>>(seed, n, table, (uint32_t *)d_bases, (uint64_t *)d_b);
    AB_LAUNCHED();
    return 0;
}

int gen_bases_dispatch(int curve, uint64_t seed, size_t n, void *d_bases, void *d_b, cudaStream_t st) {
    if (!d_bases && n) { set_last_error("null pointer"); return B200_EINVAL; }
    if (n == 0) return 0;
    if (curve == B200_CURVE_BLS12_381) return gen_bases_run<GenG1<BlsFq>>(curve, seed, n, d_bases, d_b, st);
    if (curve == B200_CURVE_BN254) return gen_bases_run<GenG1<BnFq>>(curve, seed, n, d_bases, d_b, st);
    if (curve == B200_CURVE_BLS12_381_G2) return gen_bases_run<GenBlsG2>(curve, seed, n, d_bases, d_b, st);
    set_last_error("unknown curve id");
    return B200_EINVAL;
}
int gen_scalars_dispatch(int field, uint64_t seed, size_t n, void *d_scalars, cudaStream_t st) {
    if (!d_scalars && n) { set_last_error("null pointer"); return B200_EINVAL; }
    if (n == 0) return 0;
    unsigned blocks = (unsigned)((n + 255) / 256);
    if (field == B200_FIELD_BLS12_381_FR) gen_scalars_kernel<BlsFr><<<blocks, 256, 0, st>>>(seed, n, (uint32_t *)d_scalars);
    else if (field == B200_FIELD_BN254_FR) gen_scalars_kernel<BnFr><<<blocks, 256, 0, st>>>(seed, n, (uint32_t *)d_scalars);
    else { set_last_error("unknown scalar field id"); return B200_EINVAL; }
    AB_LAUNCHED();
    return 0;
}

template <class PQ, class PR> static int batch_mul_run(const uint64_t *base_xy, const void *d_scalars, size_t n, void *d_out, cudaStream_t st) {
    constexpr int L = PQ::L;
    const int windows = (PR::BITS + 7) / 8;
    LimbArg<L> bx, by;
    for (int i = 0; i < L / 2; i++) {
        bx.v[2 * i] = (uint32_t)base_xy[i]; bx.v[2 * i + 1] = (uint32_t)(base_xy[i] >> 32);
        by.v[2 * i] = (uint32_t)base_xy[L / 2 + i]; by.v[2 * i + 1] = (uint32_t)(base_xy[L / 2 + i] >> 32);
    }
    uint32_t *table = nullptr;
    AB_CUDA(cudaMallocAsync(&table, (size_t)windows * 256 * 2 * L * 4, st));
    batch_table_kernel<PQ><<<(windows * 256 + 63) / 64, 64, 0, st>>>(bx, by, windows, table);
    AB_LAUNCHED();
    size_t threads = (n + kGenBatch - 1) / kGenBatch;
    batch_mul_kernel<PQ, PR><<<(unsigned)((threads + 63) / 64), 64, 0, st>>>((const uint32_t *)d_scalars, n, table, windows, (uint32_t *)d_out);
    AB_LAUNCHED();
    AB_CUDA(cudaFreeAsync(table, st));
    return 0;
}
int batch_mul_dispatch(int curve, const uint64_t *base_xy, const void *d_scalars, size_t n, void *d_out, cudaStream_t st) {
    if (!base_xy || (n && (!d_scalars || !d_out))) { set_last_error("null pointer"); return B200_EINVAL; }
    if (n == 0) return 0;
    if (curve == B200_CURVE_BLS12_381) return batch_mul_run<BlsFq, BlsFr>(base_xy, d_scalars, n, d_out, st);
    if (curve == B200_CURVE_BN254) return batch_mul_run<BnFq, BnFr>(base_xy, d_scalars, n, d_out, st);
    set_last_error("unknown curve id");
    return B200_EINVAL;
}
int normalize_batch_dispatch(int curve, const void *d_xyz, size_t n, void *d_out, cudaStream_t st) {
    if (n && (!d_xyz || !d_out)) { set_last_error("null pointer"); return B200_EINVAL; }
    if (n == 0) return 0;
    size_t threads = (n + kGenBatch - 1) / kGenBatch;
    if (curve == B200_CURVE_BLS12_381) normalize_batch_kernel<BlsFq><<<(unsigned)((threads + 63) / 64), 64, 0, st>>>((const uint32_t *)d_xyz, n, (uint32_t *)d_out);
    else if (curve == B200_CURVE_BN254) normalize_batch_kernel<BnFq><<<(unsigned)((threads + 63) / 64), 64, 0, st>>>((const uint32_t *)d_xyz, n, (uint32_t *)d_out);
    else { set_last_error("unknown curve id"); return B200_EINVAL; }
    AB_LAUNCHED();
    return 0;
}

}  // namespace ab200
