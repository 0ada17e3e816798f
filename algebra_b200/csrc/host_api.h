// host_api.h — the library's internal host interface: every function capi.cu calls in another unit, declared once.  Each unit
// that defines one of them includes this header, so the compiler checks the definition against the declaration.
// Host-only: the device headers (fp.cuh, ec.cuh, common.cuh, msm_common.cuh) must not include it.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>

namespace ab200 {

// Facts of a public curve / scalar-field id, taken from the parameter packs; null for an unknown id.
struct CurveInfo {
    int coord_words;    // 32-bit words per coordinate (12 / 8 / 24)
    int scalar_bits;    // Fr::MODULUS_BIT_SIZE
    int scalar_field;   // B200_FIELD_* id of the curve's scalar field
};
struct FieldInfo {
    int two_adicity;
    int fp_op_field;    // field id of b200_fp_op_dev
};
const CurveInfo *curve_info(int curve);
const FieldInfo *field_info(int field);

// msm.cu
struct MsmSessionBase {
    virtual ~MsmSessionBase() {}
    // n_total: expected total number of pairs (window choice); max_chunk: largest chunk handed to add_chunk
    virtual int begin(size_t n_total, size_t max_chunk, int kind, cudaStream_t st) = 0;
    // digit-sort + accumulate one chunk into the session's buckets; `ready` (may be null) is waited on first.  Asynchronous.
    virtual int add_chunk(const void *d_bases, const void *d_scalars, size_t nk, cudaEvent_t ready) = 0;
    // bucket reduction + window combine -> d_out (3 coordinates, Jacobian).  Asynchronous on the session's stream.
    virtual int finish(void *d_out) = 0;
    // after the stream has been synchronised: fold the per-phase events into the thread's "last timings"
    virtual int collect_timings() = 0;
    virtual int coord_words() const = 0;   // 32-bit words per coordinate (12 / 8 / 24)
};
MsmSessionBase *msm_session_create(int curve);
// finish + D2H of the 3 coordinates to out_xyz on st, then synchronise st (error paths included) and collect the timings
int msm_session_result(MsmSessionBase &s, uint64_t *out_xyz, cudaStream_t st);
void msm_write_zero(int curve, uint64_t *out_xyz);
int msm_dispatch(int curve, int kind, const void *d_bases, const void *d_scalars, size_t n, uint64_t *out_xyz_host, cudaStream_t st, int K,
                 const size_t *chunk_off, const cudaEvent_t *ready);
int check_scalar_kind(int kind);
size_t scalar_kind_bytes(int kind);
int msm_set_window(int c);
int msm_set_affine_levels(int levels);
int msm_get_window();
int msm_get_affine_levels();
int msm_set_bucket_slice(int slice, int slices);
void msm_get_bucket_slice(int *slice, int *slices);
int msm_auto_window(size_t n, int scalar_bits);
int msm_last_timings(float *ms7, int *c, int *windows, unsigned long long *bucket_adds);
// sum of k Jacobian points (to_affine: the affine form of each of the k points), device buffers, asynchronous on st
int g1_sum(int curve, const void *d_pts, size_t k, void *d_out, bool to_affine, cudaStream_t st);

// ntt.cu, point_ntt.cu
int ntt_dispatch(int field, void *d_data, uint32_t log_n, int inverse, const uint64_t *coset, cudaStream_t st);
int ntt_clear_cache();
int point_ntt_check(int curve, const void *points, uint32_t log_n);
int point_ntt_dispatch(int curve, void *d_points, uint32_t log_n, int inverse, const uint64_t *coset, cudaStream_t st);

// prims.cu, gen.cu
int fp_op_dispatch(int field, int op, const void *a, const void *b, void *out, size_t n, int reps, cudaStream_t st);
int ec_op_dispatch(int curve, int op, const void *a, const void *b, void *out, size_t n, cudaStream_t st);
int gen_bases_dispatch(int curve, uint64_t seed, size_t n, void *d_bases, void *d_b, cudaStream_t st);
int gen_scalars_dispatch(int field, uint64_t seed, size_t n, void *d_scalars, cudaStream_t st);
int batch_mul_dispatch(int curve, const uint64_t *base_xy, const void *d_scalars, size_t n, void *d_out, cudaStream_t st);
int normalize_batch_dispatch(int curve, const void *d_xyz, size_t n, void *d_out, cudaStream_t st);

}  // namespace ab200
