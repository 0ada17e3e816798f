// prims.cu — element-wise kernels over the device arithmetic headers (1 thread per element): the parity surface for
// fp.cuh / ec.cuh on the real GPU and the field micro-benchmark (cf. bench-templates/src/macros/field.rs:69-155).
#include "common.cuh"
#include "host_api.h"
#include "ec.cuh"

namespace ab200 {

template <class P> __global__ void fp_op_kernel(int op, const uint32_t *a, const uint32_t *b, uint32_t *out, size_t n, int reps) {
    using F = Fp<P>;
    constexpr int L = P::L;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t x[L], y[L], r[L];
    load_limbs<L>(x, a + i * L);
    if (b) load_limbs<L>(y, b + i * L);
    else limbs_copy<L>(y, x);
    for (int k = 0; k < reps; k++) {
        switch (op) {
            case 0: F::mul(r, x, y); break;
            case 1: F::add(r, x, y); break;
            case 2: F::sub(r, x, y); break;
            case 3: F::sqr(r, x); break;
            case 4: F::dbl(r, x); break;
            case 5: F::neg(r, x); break;
            case 6: F::from_mont(r, x); break;
            case 7: F::to_mont(r, x); break;
            default: F::inv(r, x); break;
        }
        limbs_copy<L>(x, r);
    }
    store_limbs<L>(out + i * L, r);
}

// same surface for the quadratic extension (field id 4 = BLS12-381 Fq2): ops 0 mul 1 add 2 sub 3 square 4 double 5 neg 8 inverse
template <class F> __global__ void fp2_op_kernel(int op, const uint32_t *a, const uint32_t *b, uint32_t *out, size_t n, int reps) {
    constexpr int L = F::L;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t x[L], y[L], r[L];
    load_limbs<L>(x, a + i * L);
    if (b) load_limbs<L>(y, b + i * L);
    else limbs_copy<L>(y, x);
    for (int k = 0; k < reps; k++) {
        switch (op) {
            case 0: F::mul(r, x, y); break;
            case 1: F::add(r, x, y); break;
            case 2: F::sub(r, x, y); break;
            case 3: F::sqr(r, x); break;
            case 4: F::dbl(r, x); break;
            case 5: F::neg(r, x); break;
            default: F::inv(r, x); break;
        }
        limbs_copy<L>(x, r);
    }
    store_limbs<L>(out + i * L, r);
}

template <class FT> __global__ void ec_op_kernel(int op, const uint32_t *a, const uint32_t *b, uint32_t *out, size_t n) {
    using E = Ec<FT>;
    constexpr int L = FT::L;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    typename E::B x, y;
    typename E::J j, k;
    if (op <= 4) {
        const uint32_t *p = a + i * 4 * L;
        load_limbs<L>(x.x, p); load_limbs<L>(x.y, p + L); load_limbs<L>(x.zz, p + 2 * L); load_limbs<L>(x.zzz, p + 3 * L);
    } else {
        const uint32_t *p = a + i * 3 * L;
        load_limbs<L>(j.x, p); load_limbs<L>(j.y, p + L); load_limbs<L>(j.z, p + 2 * L);
    }
    if (op == 0 || op == 1) {
        uint32_t px[L], py[L];
        load_limbs<L>(px, b + i * 2 * L); load_limbs<L>(py, b + i * 2 * L + L);
        E::madd(x, px, py, op == 1);
    } else if (op == 2) {
        const uint32_t *p = b + i * 4 * L;
        load_limbs<L>(y.x, p); load_limbs<L>(y.y, p + L); load_limbs<L>(y.zz, p + 2 * L); load_limbs<L>(y.zzz, p + 3 * L);
        E::xyzz_add(x, y);
    } else if (op == 3) {
        E::xyzz_dbl(x);
    } else if (op == 4) {
        E::xyzz_to_jac(j, x);
    } else if (op == 5) {
        uint32_t ax[L], ay[L];
        E::jac_to_affine(ax, ay, j);
        store_limbs<L>(out + i * 2 * L, ax); store_limbs<L>(out + i * 2 * L + L, ay);
        return;
    } else if (op == 6) {
        const uint32_t *p = b + i * 3 * L;
        load_limbs<L>(k.x, p); load_limbs<L>(k.y, p + L); load_limbs<L>(k.z, p + 2 * L);
        E::jac_add(j, k);
    } else {
        E::jac_dbl(j);
    }
    if (op <= 3) {
        uint32_t *p = out + i * 4 * L;
        store_limbs<L>(p, x.x); store_limbs<L>(p + L, x.y); store_limbs<L>(p + 2 * L, x.zz); store_limbs<L>(p + 3 * L, x.zzz);
    } else {
        uint32_t *p = out + i * 3 * L;
        store_limbs<L>(p, j.x); store_limbs<L>(p + L, j.y); store_limbs<L>(p + 2 * L, j.z);
    }
}

int fp_op_dispatch(int field, int op, const void *a, const void *b, void *out, size_t n, int reps, cudaStream_t st) {
    if (!a || !out || op < 0 || op > 8 || reps < 1) { set_last_error("bad argument"); return B200_EINVAL; }
    if (n == 0) return 0;
    unsigned blocks = (unsigned)((n + 127) / 128);
    const uint32_t *A = (const uint32_t *)a, *B = (const uint32_t *)b;
    uint32_t *O = (uint32_t *)out;
    switch (field) {
        case 0: fp_op_kernel<BlsFq><<<blocks, 128, 0, st>>>(op, A, B, O, n, reps); break;
        case 1: fp_op_kernel<BlsFr><<<blocks, 128, 0, st>>>(op, A, B, O, n, reps); break;
        case 2: fp_op_kernel<BnFq><<<blocks, 128, 0, st>>>(op, A, B, O, n, reps); break;
        case 3: fp_op_kernel<BnFr><<<blocks, 128, 0, st>>>(op, A, B, O, n, reps); break;
        case 4:
            if (op == 6 || op == 7) { set_last_error("into/from_bigint are not defined for Fq2"); return B200_EINVAL; }
            fp2_op_kernel<Fp2<BlsFq>><<<blocks, 128, 0, st>>>(op, A, B, O, n, reps);
            break;
        default: set_last_error("unknown field id"); return B200_EINVAL;
    }
    AB_LAUNCHED();
    return 0;
}
int ec_op_dispatch(int curve, int op, const void *a, const void *b, void *out, size_t n, cudaStream_t st) {
    if (!a || !out || op < 0 || op > 7) { set_last_error("bad argument"); return B200_EINVAL; }
    if ((op == 0 || op == 1 || op == 2 || op == 6) && !b) { set_last_error("second operand required"); return B200_EINVAL; }
    if (n == 0) return 0;
    unsigned blocks = (unsigned)((n + 63) / 64);
    if (curve == B200_CURVE_BLS12_381) ec_op_kernel<Fp<BlsFq>><<<blocks, 64, 0, st>>>(op, (const uint32_t *)a, (const uint32_t *)b, (uint32_t *)out, n);
    else if (curve == B200_CURVE_BN254) ec_op_kernel<Fp<BnFq>><<<blocks, 64, 0, st>>>(op, (const uint32_t *)a, (const uint32_t *)b, (uint32_t *)out, n);
    else if (curve == B200_CURVE_BLS12_381_G2) ec_op_kernel<Fp2<BlsFq>><<<blocks, 64, 0, st>>>(op, (const uint32_t *)a, (const uint32_t *)b, (uint32_t *)out, n);
    else { set_last_error("unknown curve id"); return B200_EINVAL; }
    AB_LAUNCHED();
    return 0;
}

}  // namespace ab200
