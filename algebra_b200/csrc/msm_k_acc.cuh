// msm_k_acc.cuh — digit extraction, task-balanced XYZZ accumulation, fix-ups, bucket merge, and their launchers.
#pragma once
#include "msm_common.cuh"

namespace ab200 {

// ------------------------------------------------------------------------------------------------
// digits: canonical scalar -> signed digits (make_digits, :754-794), every window's digit written once, window-major:
// digits[w * n + i] = rel | sign << 31 (rel = bucket inside the window's slice) or kNoDigit — the input of the bucket sort
// ------------------------------------------------------------------------------------------------
template <class C>
__global__ void __launch_bounds__(256) msm_digits_kernel(const void *__restrict__ scalars_v, int kind, size_t n, MsmGeom g,
                                                         uint32_t *__restrict__ digits) {
    using FR = Fp<typename C::Fr>;
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t k[10];
#pragma unroll
    for (int j = 0; j < 10; j++) k[j] = 0;
    if (kind <= B200_SCALARS_BIGINT) {
        uint32_t s[8];
        load_limbs_nc<8>(s, (const uint32_t *)scalars_v + i * 8);
        if (kind == B200_SCALARS_FR_MONT) FR::from_mont(k, s);  // into_bigint (:60-62)
        else limbs_copy<8>(k, s);                               // msm_bigint: already canonical (:80-85)
    } else if (kind == B200_SCALARS_U8) k[0] = ((const uint8_t *)scalars_v)[i];
    else if (kind == B200_SCALARS_U16) k[0] = ((const uint16_t *)scalars_v)[i];
    else if (kind == B200_SCALARS_U32) k[0] = ((const uint32_t *)scalars_v)[i];
    else { uint2 v = ((const uint2 *)scalars_v)[i]; k[0] = v.x; k[1] = v.y; }
    // msm_signed's negative classes (variable_base/mod.rs:251-336): a scalar whose r - k fits 64 bits (NegU1..NegU64) is
    // handled as -(r - k), i.e. the point enters with the opposite sign and only ceil(64/c) windows are non-zero
    uint32_t flip = 0;
    if (kind <= B200_SCALARS_BIGINT && (k[2] | k[3] | k[4] | k[5] | k[6] | k[7])) {
        using R = typename C::Fr;
        uint32_t t[8];
        t[0] = ptx::sub_cc(R::MOD(0), k[0]);
#pragma unroll
        for (int j = 1; j < 8; j++) t[j] = ptx::subc_cc(R::MOD(j), k[j]);
        const uint32_t borrow = ptx::subc(0u, 0u);   // non-zero iff k > r (non-canonical msm_bigint input: left alone)
        if (!borrow && !(t[2] | t[3] | t[4] | t[5] | t[6] | t[7])) {
#pragma unroll
            for (int j = 0; j < 8; j++) k[j] = t[j];
            flip = 1;
        }
    }
    const int c = g.c;
    const uint32_t mask = (1u << c) - 1, half = 1u << (c - 1);
    uint32_t carry = 0;
    for (int w = 0; w < g.W; w++) {
        const int bit = w * c, wi = bit >> 5, sh = bit & 31;
        uint64_t two = ((uint64_t)k[wi + 1] << 32) | k[wi];
        uint32_t coef = ((uint32_t)(two >> sh) & mask) + carry;
        uint32_t mag, neg = 0;
        if (w == g.W - 1) {  // top digit stays unsigned (:789-791); bits above the declared scalar width are ignored
            mag = (((uint32_t)(two >> sh) & mask) & ((1u << g.top_bits) - 1)) + carry;
        } else {
            carry = (coef + half) >> c;
            if (carry) { mag = (1u << c) - coef; neg = 1; }  // digit = coef - 2^c in [-2^(c-1), 0)
            else mag = coef;
        }
        // bucket slice: only the magnitudes in [off, off + nbw) of each window belong to this session (whole window by default)
        const uint32_t rel = mag - 1 - ((w == g.W - 1) ? g.off_top : g.off);
        const bool keep = mag && rel < ((w == g.W - 1) ? g.nb_top : g.nb);
        digits[(size_t)w * n + i] = keep ? rel | ((neg ^ flip) << 31) : kNoDigit;
    }
}
// ------------------------------------------------------------------------------------------------
// bucket accumulation — the hot loop (Bucket += Affine, bucket.rs:168-238), balanced by construction:
// the bucket-sorted entry array is cut into tasks of exactly T consecutive entries, one thread per task, whatever the
// bucket sizes are (a scalar distribution that piles everything into one bucket, or a short top window with 8 buckets
// holding n/8 points each, costs the same as the uniform case).  A thread walks its slice and flushes an accumulator at
// every bucket boundary: buckets that begin and end inside the slice are written straight to `buckets`; the piece of a
// bucket that began in an earlier task goes to head[t], the piece of a bucket that continues into the next task to tail[t].
// msm_fixup_* then add tail[t0] + head[t0+1..t1] for every bucket that spans tasks.  `buckets` is pre-zeroed (zz = zzz = 0
// is the XYZZ identity) so empty buckets need no writer.
// ------------------------------------------------------------------------------------------------

template <int L> __device__ __forceinline__ void store_xyzz(uint32_t *p, const Xyzz<L> &b);
template <int L> __device__ __forceinline__ void load_xyzz(Xyzz<L> &b, const uint32_t *p);

// DIRECT = false: entry p is `sorted[p]` = (base index | sign<<31), gathered from `bases`;
// DIRECT = true : entry p is the affine point stored at bases[p] (output of the batched-affine pre-reduction), no sign.
template <class C, bool DIRECT>
__global__ void __launch_bounds__(128) msm_accumulate_kernel(const uint32_t *__restrict__ bases, const uint32_t *__restrict__ sorted,
                                                             const uint32_t *__restrict__ offsets, uint32_t total_buckets, uint32_t T,
                                                             uint32_t *__restrict__ buckets, uint32_t *__restrict__ head,
                                                             uint32_t *__restrict__ tail, uint32_t *__restrict__ head_bucket,
                                                             uint32_t *__restrict__ tail_bucket, uint32_t num_tasks) {
    using F = typename C::F;
    using E = Ec<F>;
    constexpr int L = F::L;
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= num_tasks) return;
    // `offsets` may be a window group's slice of a larger offsets array: entry positions start at offsets[0]
    const uint32_t M = __ldg(offsets + total_buckets);
    const uint64_t lo64 = (uint64_t)__ldg(offsets) + (uint64_t)t * T;
    if (lo64 >= M) {
        head_bucket[t] = kNoBucket;
        tail_bucket[t] = kNoBucket;
        return;
    }
    const uint32_t lo = (uint32_t)lo64, hi = (uint32_t)min((uint64_t)M, lo64 + T);
    // b = last index with offsets[b] <= lo  (=> offsets[b] <= lo < offsets[b+1])
    uint32_t bl = 0, br = total_buckets;  // invariant: offsets[bl] <= lo, offsets[br] > lo (offsets[total] = M > lo)
    while (br - bl > 1) {
        uint32_t mid = bl + ((br - bl) >> 1);
        if (__ldg(offsets + mid) <= lo) bl = mid; else br = mid;
    }
    uint32_t b = bl, bucket_end = __ldg(offsets + b + 1);
    bool started_before = __ldg(offsets + b) < lo;
    uint32_t hb = kNoBucket;

    typename E::B acc;
    E::xyzz_set_zero(acc);
    uint32_t cx[L], cy[L], nx[L], ny[L];
    uint32_t e = DIRECT ? lo : __ldg(sorted + lo), e_next = 0;
    {
        const uint32_t *bp = bases + (size_t)(DIRECT ? e : (e & 0x7fffffffu)) * (2 * L);
        load_limbs_nc<L>(cx, bp);
        load_limbs_nc<L>(cy, bp + L);
    }
    for (uint32_t pos = lo; pos < hi; pos++) {
        const bool more = (pos + 1 < hi);
        if (more) {  // issue the next gather before the ~10 modmuls of this addition
            e_next = DIRECT ? pos + 1 : __ldg(sorted + pos + 1);
            const uint32_t *bp = bases + (size_t)(DIRECT ? e_next : (e_next & 0x7fffffffu)) * (2 * L);
            load_limbs_nc<L>(nx, bp);
            load_limbs_nc<L>(ny, bp + L);
        }
        if (pos == bucket_end) {  // bucket b is complete: flush, move to the (non-empty) bucket that owns `pos`
            if (started_before) { store_xyzz<L>(head + (size_t)t * (4 * L), acc); hb = b; }
            else store_xyzz<L>(buckets + (size_t)b * (4 * L), acc);
            E::xyzz_set_zero(acc);
            started_before = false;
            do { b++; bucket_end = __ldg(offsets + b + 1); } while (bucket_end <= pos);
        }
        E::madd(acc, cx, cy, !DIRECT && (e >> 31) != 0);
        if (more) {
            limbs_copy<L>(cx, nx);
            limbs_copy<L>(cy, ny);
            e = e_next;
        }
    }
    uint32_t tb = kNoBucket;
    if (bucket_end == hi) {  // the last bucket ends exactly with the slice
        if (started_before) { store_xyzz<L>(head + (size_t)t * (4 * L), acc); hb = b; }
        else store_xyzz<L>(buckets + (size_t)b * (4 * L), acc);
    } else if (started_before) {  // the whole slice is an inner piece of one bucket
        store_xyzz<L>(head + (size_t)t * (4 * L), acc);
        hb = b;
    } else {
        store_xyzz<L>(tail + (size_t)t * (4 * L), acc);
        tb = b;
    }
    head_bucket[t] = hb;
    tail_bucket[t] = tb;
}
// small spans: one thread per task boundary; long spans (heavy buckets): one block per bucket.
template <class C>
__global__ void __launch_bounds__(128) msm_fixup_small_kernel(const uint32_t *__restrict__ offsets, uint32_t T, const uint32_t *__restrict__ head,
                                                              const uint32_t *__restrict__ tail, const uint32_t *__restrict__ tail_bucket,
                                                              uint32_t num_tasks, uint32_t *__restrict__ buckets) {
    using F = typename C::F;
    using E = Ec<F>;
    constexpr int L = F::L;
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= num_tasks) return;
    const uint32_t b = tail_bucket[t];
    if (b == kNoBucket) return;
    const uint32_t t1 = (__ldg(offsets + b + 1) - 1 - __ldg(offsets)) / T;
    if (t1 - t > kFixupSmall) return;
    typename E::B acc, x;
    load_xyzz<L>(acc, tail + (size_t)t * (4 * L));
    for (uint32_t k = t + 1; k <= t1; k++) {
        load_xyzz<L>(x, head + (size_t)k * (4 * L));
        E::xyzz_add(acc, x);
    }
    store_xyzz<L>(buckets + (size_t)b * (4 * L), acc);
}
template <class C>
__global__ void __launch_bounds__(128) msm_fixup_big_kernel(const uint32_t *__restrict__ offsets, uint32_t T, const uint32_t *__restrict__ head,
                                                            const uint32_t *__restrict__ tail, const uint32_t *__restrict__ tail_bucket,
                                                            uint32_t num_tasks, uint32_t *__restrict__ buckets) {
    using F = typename C::F;
    using E = Ec<F>;
    constexpr int L = F::L;
    extern __shared__ uint32_t sm[];
    const uint32_t t = blockIdx.x;
    if (t >= num_tasks) return;
    const uint32_t b = tail_bucket[t];
    if (b == kNoBucket) return;
    const uint32_t t1 = (__ldg(offsets + b + 1) - 1 - __ldg(offsets)) / T;
    if (t1 - t <= kFixupSmall) return;
    typename E::B acc, x;
    E::xyzz_set_zero(acc);
    if (threadIdx.x == 0) load_xyzz<L>(acc, tail + (size_t)t * (4 * L));
    for (uint32_t k = t + 1 + threadIdx.x; k <= t1; k += blockDim.x) {
        load_xyzz<L>(x, head + (size_t)k * (4 * L));
        E::xyzz_add(acc, x);
    }
    store_xyzz<L>(sm + threadIdx.x * (4 * L), acc);
    __syncthreads();
    for (uint32_t s2 = blockDim.x >> 1; s2 > 0; s2 >>= 1) {
        if (threadIdx.x < s2) {
            load_xyzz<L>(acc, sm + threadIdx.x * (4 * L));
            load_xyzz<L>(x, sm + (threadIdx.x + s2) * (4 * L));
            E::xyzz_add(acc, x);
            store_xyzz<L>(sm + threadIdx.x * (4 * L), acc);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        load_xyzz<L>(acc, sm);
        store_xyzz<L>(buckets + (size_t)b * (4 * L), acc);
    }
}
// buckets[b] += extra[b]  (chunked paths: every chunk after the first accumulates into `extra`)
template <class C>
__global__ void __launch_bounds__(128) msm_merge_kernel(uint32_t *__restrict__ buckets, const uint32_t *__restrict__ extra, uint32_t total_buckets) {
    using F = typename C::F;
    using E = Ec<F>;
    constexpr int L = F::L;
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= total_buckets) return;
    typename E::B x, y;
    load_xyzz<L>(y, extra + (size_t)b * (4 * L));
    if (E::xyzz_is_zero(y)) return;
    load_xyzz<L>(x, buckets + (size_t)b * (4 * L));
    E::xyzz_add(x, y);
    store_xyzz<L>(buckets + (size_t)b * (4 * L), x);
}


template <class C> int MsmAccLaunch<C>::digits(const void *scalars, int kind, size_t nk, MsmGeom g, uint32_t *digits, cudaStream_t st) {
    msm_digits_kernel<C><<<(unsigned)((nk + 255) / 256), 256, 0, st>>>(scalars, kind, nk, g, digits);
    AB_LAUNCHED();
    return 0;
}
template <class C> int MsmAccLaunch<C>::occupancy(bool direct) {
    int b = 0;
    cudaError_t e = direct ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, msm_accumulate_kernel<C, true>, 128, 0)
                           : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, msm_accumulate_kernel<C, false>, 128, 0);
    return (e == cudaSuccess && b > 0) ? b : 2;
}
template <class C>
int MsmAccLaunch<C>::accumulate(bool direct, const uint32_t *pts, const uint32_t *sorted_idx, const uint32_t *offs, uint32_t nbk, uint32_t T,
                                uint32_t num_tasks, uint32_t *dst, uint32_t *head, uint32_t *tail, uint32_t *head_bucket, uint32_t *tail_bucket,
                                cudaStream_t st) {
    constexpr int L = C::F::L;
    const unsigned grid = (num_tasks + 127) / 128;
    if (direct) msm_accumulate_kernel<C, true><<<grid, 128, 0, st>>>(pts, nullptr, offs, nbk, T, dst, head, tail, head_bucket, tail_bucket, num_tasks);
    else msm_accumulate_kernel<C, false><<<grid, 128, 0, st>>>(pts, sorted_idx, offs, nbk, T, dst, head, tail, head_bucket, tail_bucket, num_tasks);
    AB_LAUNCHED();
    msm_fixup_small_kernel<C><<<grid, 128, 0, st>>>(offs, T, head, tail, tail_bucket, num_tasks, dst);
    AB_LAUNCHED();
    AB_CUDA(cudaFuncSetAttribute(msm_fixup_big_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 4 * L * 4));
    msm_fixup_big_kernel<C><<<num_tasks, 128, 128 * 4 * L * 4, st>>>(offs, T, head, tail, tail_bucket, num_tasks, dst);
    AB_LAUNCHED();
    return 0;
}
template <class C> int MsmAccLaunch<C>::merge(uint32_t *buckets, const uint32_t *extra, uint32_t nb, cudaStream_t st) {
    msm_merge_kernel<C><<<(nb + 127) / 128, 128, 0, st>>>(buckets, extra, nb);
    AB_LAUNCHED();
    return 0;
}

}  // namespace ab200
