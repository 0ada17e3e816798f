// msm.cu — variable-base MSM over short-Weierstrass G1 (a = 0) for sm_90a: bucket method (Pippenger) with signed c-bit
// digits, counting-sort bucket assignment, batched-affine pre-reduction and task-balanced XYZZ accumulation.
//
// Replaces VariableBaseMSM::msm_unchecked for Projective<P> (ec/src/scalar_mul/variable_base/mod.rs:59-64
// -> msm_bigint_wnaf_parallel :437-503).  Same mathematics, GPU schedule:
//   reference (per window, serial over points)          here (all windows at once)
//   into_bigint + make_digits (:60-62, :754-794)    ->  msm_digits_kernel: REDC + signed digits of every window, written once
//   buckets[|d|-1] +=/-= base  (:467-475)           ->  msm_sort.cu: two-pass counting sort (coarse bins, then each bin in shared
//                                                       memory) into (index | sign) in bucket order;
//                                                       msm_pairmap_kernel + msm_pair_add_kernel x up to 4 levels: every bucket run
//                                                       is halved with AFFINE additions that share one inversion per block
//                                                       (Montgomery's trick);
//                                                       msm_accumulate_kernel: one thread per task of T entries runs the reference's
//                                                       `Bucket += Affine` (bucket.rs:168-238) on what is left, flushing per bucket;
//                                                       msm_fixup_*: buckets that span tasks
//   running-sum  res += running_sum (:478-484)      ->  msm_bucket_reduce_kernel (running sum per chunk of 32 buckets + chunk offset times
//                                                       chunk total) and msm_sum_partials_kernel (tree over the chunks of a window)
//   window combine, c doublings per window (:489-502) -> msm_window_combine_coop_kernel (Jacobian, one warp)
// EC addition is commutative/associative, so bucket order, atomics, pairing and chunking do not change the group element;
// results are compared with the reference after into_affine(), limb-exact.
// The digit recoding is the reference's make_digits (top window unsigned), so bucket counts per window are 2^(c-1), and
// 2^(lambda-(W-1)c) for the top window.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <memory>
#include <vector>

#include "host_api.h"
#include "msm_common.cuh"

namespace ab200 {

// ------------------------------------------------------------------------------------------------
// exclusive scan of u32 counts (total < 2^32): block totals -> serial scan of totals -> apply
// ------------------------------------------------------------------------------------------------
static constexpr int kScanThreads = 512, kScanPerThread = 8, kScanBlock = kScanThreads * kScanPerThread;

__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t *total) {
    __shared__ uint32_t warp_sums[32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[wid] = x;
    __syncthreads();
    if (wid == 0) {
        uint32_t ws = (lane < (int)(blockDim.x >> 5)) ? warp_sums[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            uint32_t y = __shfl_up_sync(0xffffffffu, ws, o);
            if (lane >= o) ws += y;
        }
        warp_sums[lane] = ws;  // inclusive
    }
    __syncthreads();
    uint32_t before = wid ? warp_sums[wid - 1] : 0;
    *total = warp_sums[(blockDim.x >> 5) - 1];
    return before + x - v;  // exclusive
}

__global__ void __launch_bounds__(kScanThreads) scan_block_totals_kernel(const uint32_t *in, size_t n, uint32_t *block_totals) {
    size_t base = (size_t)blockIdx.x * kScanBlock + (size_t)threadIdx.x * kScanPerThread;
    uint32_t s = 0;
#pragma unroll
    for (int k = 0; k < kScanPerThread; k++)
        if (base + k < n) s += in[base + k];
    uint32_t total;
    block_exclusive_scan(s, &total);
    if (threadIdx.x == 0) block_totals[blockIdx.x] = total;
}
__global__ void __launch_bounds__(kScanThreads) scan_totals_kernel(uint32_t *block_totals, size_t nblocks) {
    __shared__ uint32_t running;
    if (threadIdx.x == 0) running = 0;
    __syncthreads();
    for (size_t base = 0; base < nblocks; base += kScanThreads) {
        size_t i = base + threadIdx.x;
        uint32_t v = i < nblocks ? block_totals[i] : 0, total;
        uint32_t ex = block_exclusive_scan(v, &total);
        uint32_t r0 = running;
        if (i < nblocks) block_totals[i] = r0 + ex;
        __syncthreads();
        if (threadIdx.x == 0) running = r0 + total;
        __syncthreads();
    }
}
// out[i] = exclusive prefix; out[n] = grand total (out has n+1 entries)
__global__ void __launch_bounds__(kScanThreads) scan_apply_kernel(const uint32_t *in, size_t n, const uint32_t *block_offsets, uint32_t *out) {
    size_t base = (size_t)blockIdx.x * kScanBlock + (size_t)threadIdx.x * kScanPerThread;
    uint32_t v[kScanPerThread], s = 0;
#pragma unroll
    for (int k = 0; k < kScanPerThread; k++) {
        v[k] = (base + k < n) ? in[base + k] : 0;
        s += v[k];
    }
    uint32_t total;
    uint32_t ex = block_exclusive_scan(s, &total) + block_offsets[blockIdx.x];
#pragma unroll
    for (int k = 0; k < kScanPerThread; k++) {
        if (base + k < n) out[base + k] = ex;
        ex += v[k];
        if (base + k == n - 1) out[n] = ex;
    }
}
// ------------------------------------------------------------------------------------------------
// Batched-affine pre-reduction (optional stage between the sort and the XYZZ accumulation).
// One level halves every bucket's run: output slot j of bucket b = in[2j] + in[2j+1] (or in[2j] alone when the run is odd),
// as AFFINE points.  Affine addition needs 1/(x2 - x1); a thread owns `batch` output slots and the 128 threads of a block
// invert all their denominators with ONE field inversion (Montgomery's trick: forward pass stores the running products in
// the output slots themselves, backward pass peels them off) — ~6 modmuls + inversion/(128 batch) per addition instead of
// the 10 of an XYZZ mixed addition.  Degenerate pairs keep the batch intact with a denominator of 1: an identity operand passes
// the other one through, equal points are doubled (denominator 2y), opposite points give the identity (0,0).
// Same group element as the reference's bucket sums (EC addition is associative); parity is checked after into_affine().
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) msm_halve_counts_kernel(const uint32_t *__restrict__ offsets_in, uint32_t total_buckets,
                                                               uint32_t *__restrict__ counts_out) {
    uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= total_buckets) return;
    uint32_t cnt = offsets_in[b + 1] - offsets_in[b];
    counts_out[b] = (cnt + 1) >> 1;
}
// pairmap[p] = (index of the first input entry of output slot p) | (the slot has a second entry) << 31.
// One block per 1024 consecutive slots: two threads locate the first and last bucket of the block's slot range, the bucket
// offsets in between are staged in shared memory and every slot finds its bucket by a short binary search there (any bucket
// size distribution costs the same; a run of > 2048 buckets inside one block — mostly empty ones — falls back to global loads).
__global__ void __launch_bounds__(256) msm_pairmap_kernel(const uint32_t *__restrict__ offsets_in, const uint32_t *__restrict__ offsets_out,
                                                          uint32_t nb, uint32_t *__restrict__ pairmap) {
    constexpr uint32_t SPAN = 2048;
    __shared__ uint32_t s_off[SPAN + 1];
    __shared__ uint32_t s_b[2];
    const uint32_t M = __ldg(offsets_out + nb);
    const uint64_t P0l = (uint64_t)blockIdx.x * 1024;
    if (P0l >= M) return;
    const uint32_t P0 = (uint32_t)P0l, P1 = (uint32_t)min((uint64_t)M, P0l + 1024) - 1;
    if (threadIdx.x < 2) {
        const uint32_t p = threadIdx.x ? P1 : P0;
        uint32_t lo = 0, hi = nb;   // offsets_out[lo] <= p < offsets_out[hi]
        while (hi - lo > 1) {
            const uint32_t mid = lo + ((hi - lo) >> 1);
            if (__ldg(offsets_out + mid) <= p) lo = mid; else hi = mid;
        }
        s_b[threadIdx.x] = lo;
    }
    __syncthreads();
    const uint32_t b_first = s_b[0], span = s_b[1] - s_b[0] + 1;
    const bool staged = span <= SPAN;
    if (staged)
        for (uint32_t i = threadIdx.x; i <= span; i += 256) s_off[i] = __ldg(offsets_out + b_first + i);
    __syncthreads();
    for (uint32_t q = threadIdx.x; q < 1024; q += 256) {
        const uint32_t p = P0 + q;
        if (p > P1) break;
        uint32_t lo = 0, hi = span;   // off[lo] <= p < off[hi]
        while (hi - lo > 1) {
            const uint32_t mid = lo + ((hi - lo) >> 1);
            const uint32_t v = staged ? s_off[mid] : __ldg(offsets_out + b_first + mid);
            if (v <= p) lo = mid; else hi = mid;
        }
        const uint32_t b = b_first + lo, out_beg = staged ? s_off[lo] : __ldg(offsets_out + b);
        const uint32_t in_beg = __ldg(offsets_in + b), in_end = __ldg(offsets_in + b + 1);
        const uint32_t k = in_beg + 2 * (p - out_beg);
        pairmap[p] = k | ((k + 1 < in_end) ? 0x80000000u : 0u);
    }
}
// ------------------------------------------------------------------------------------------------
// host driver
// ------------------------------------------------------------------------------------------------
// Options of a call.  Defaults come from the per-thread setters (b200_set_msm_window / _affine_levels) and, for the tuning
// knobs without a public setter, from environment variables read ONCE per process (never on the call path).
// The first MSM of the process builds EnvKnobs; changing a B200_MSM_* variable afterwards has no effect, so a test of a knob
// must set it in a fresh process before that process's first MSM (tests/test_gpu_msm_paths.py runs one child per setting).
struct EnvKnobs {
    double level_budget_bytes = 48e9;     // scratch allowed for the affine level arrays (window groups are sized to fit); also capped
                                          // by 60 % of the free device memory at the start of the call, which on an 80 GB H100 is the
                                          // binding limit for 2^26 inputs (the levels of all windows would take ~63 GB).  Fewer groups
                                          // are faster: groups shorten the batches of the later levels
    int min_batch = 96;                   // automatic mode: shortest per-thread batch a level may run with (overhead per addition:
                                          // 590/(4*batch) multiplications of the block-shared inversion)
    double level_min_load = 16.0;         // automatic mode: keep adding affine levels while the average bucket still holds this many entries
    int level_cap = 8;                    // upper bound on top of the per-curve LEVEL_CAP
    int reduce_log_m = 6;                 // buckets per reduction thread = 2^reduce_log_m at most
    bool reduce_log_m_forced = false;     // set through the environment: used as given (tuning runs)
    int force_chunks = 0;                 // test hook: split device-resident inputs into this many chunks
    EnvKnobs() {
        if (const char *e = getenv("B200_MSM_LEVEL_BUDGET_GB")) { double v = atof(e); if (v > 0.01) level_budget_bytes = v * 1e9; }
        if (const char *e = getenv("B200_MSM_MIN_BATCH")) min_batch = std::max(8, atoi(e));
        if (const char *e = getenv("B200_MSM_LEVEL_MIN_LOAD")) level_min_load = std::max(2.0, atof(e));
        if (const char *e = getenv("B200_MSM_LEVEL_CAP")) level_cap = std::min(8, std::max(0, atoi(e)));
        if (const char *e = getenv("B200_MSM_REDUCE_LOG_M")) { reduce_log_m = std::min(8, std::max(0, atoi(e))); reduce_log_m_forced = true; }
        if (const char *e = getenv("B200_MSM_FORCE_CHUNKS")) force_chunks = atoi(e);
    }
};
static const EnvKnobs &env_knobs() {
    static const EnvKnobs k;
    return k;
}

static thread_local int t_window_override = 0;
static thread_local int t_affine_levels = -1;   // batched-affine pre-reduction levels; -1 = automatic
static thread_local int t_slice = 0, t_slices = 1;   // bucket slice computed by this thread's MSMs (make_geom)
struct MsmTimings {
    float ms[7] = {0, 0, 0, 0, 0, 0, 0};
    int c = 0, W = 0;
    unsigned long long bucket_adds = 0;
};
static thread_local MsmTimings t_last;

int msm_set_affine_levels(int levels) {
    if (levels < -1 || levels > 8) { set_last_error("affine levels must be in [-1, 8]"); return B200_EINVAL; }
    t_affine_levels = levels;
    return 0;
}

int msm_set_bucket_slice(int slice, int slices) {
    if (slices < 1 || slices > 64 || slice < 0 || slice >= slices) { set_last_error("bucket slice must satisfy 0 <= slice < slices <= 64"); return B200_EINVAL; }
    t_slice = slice;
    t_slices = slices;
    return 0;
}
void msm_get_bucket_slice(int *slice, int *slices) { *slice = t_slice; *slices = t_slices; }
int msm_get_window() { return t_window_override; }
int msm_get_affine_levels() { return t_affine_levels; }
int msm_set_window(int c) {
    if (c < 0 || c > 24) { set_last_error("window size must be in [1,24] (0 = automatic)"); return B200_EINVAL; }
    t_window_override = c;
    return 0;
}

// Window choice: a relative time model of the phases (BLS12-381 G1, n = 2^22 .. 2^26): accumulation per (point, window), cheaper
//   when the average bucket holds >= ~100 entries (four affine levels) than at 32 entries per bucket (fewer levels, more XYZZ work);
//   bucket reduction per bucket; histogram + scatter per entry, + contention when the top window has fewer than ~2^10 buckets; a
//   fixed tail (reduction tree, combine).  Only the ratios of the coefficients matter for the choice of c.
int msm_auto_window(size_t n, int scalar_bits) {
    if (n < 32) return 3;  // same floor as the reference (:445-449)
    double best = 1e300;
    int best_c = 3;
    for (int c = 4; c <= 23; c++) {
        MsmGeom g = make_geom(c, scalar_bits);
        if ((double)g.total_buckets * 192.0 > 24e9) continue;
        const double entries = (double)n * g.W, load = (double)n / (double)g.nb;
        const double per = 0.28 * (1.0 + 0.8 * std::max(0.0, (100.0 - load) / 100.0));
        double t = per * entries + 2.1 * (double)g.total_buckets + 0.035 * entries;
        if (g.top_bits < 10) t += 0.25 * (double)n;   // hot top-window buckets serialise the atomics
        t += 1.5e6 + 25e3 * g.W;                       // fixed tail + per-window costs
        if (t < best) { best = t; best_c = c; }
    }
    return best_c;
}

static int scalar_kind_bits(int kind, int field_bits) {
    switch (kind) {
        case B200_SCALARS_U8: return 8;
        case B200_SCALARS_U16: return 16;
        case B200_SCALARS_U32: return 32;
        case B200_SCALARS_U64: return 64;
        default: return field_bits;  // Fr::MODULUS_BIT_SIZE (variable_base/mod.rs:451)
    }
}
int check_scalar_kind(int kind) {
    if (kind < B200_SCALARS_FR_MONT || kind > B200_SCALARS_U64) { set_last_error("unknown scalar kind"); return B200_EINVAL; }
    return 0;
}
size_t scalar_kind_bytes(int kind) {
    switch (kind) {
        case B200_SCALARS_U8: return 1;
        case B200_SCALARS_U16: return 2;
        case B200_SCALARS_U32: return 4;
        case B200_SCALARS_U64: return 8;
        default: return 32;
    }
}

// stream-ordered scratch and events owned by a session: everything is released on every exit path (cudaFreeAsync on the
// session's stream / cudaEventDestroy), including the error returns of AB_CUDA / AB_LAUNCHED.
struct StreamArena {
    cudaStream_t st = 0;
    std::vector<void *> ptrs;
    template <class T> int alloc(T **p, size_t bytes) {
        void *q = nullptr;
        AB_CUDA(cudaMallocAsync(&q, bytes ? bytes : 16, st));
        ptrs.push_back(q);
        *p = (T *)q;
        return 0;
    }
    void release(void *p) {
        if (!p) return;
        for (auto &q : ptrs)
            if (q == p) { cudaFreeAsync(q, st); q = nullptr; return; }
    }
    ~StreamArena() {
        for (void *q : ptrs)
            if (q) cudaFreeAsync(q, st);
    }
};
struct EventSet {
    std::vector<cudaEvent_t> ev;
    int make(cudaEvent_t *e) {
        AB_CUDA(cudaEventCreate(e));
        ev.push_back(*e);
        return 0;
    }
    ~EventSet() {
        for (auto e : ev) cudaEventDestroy(e);
    }
};

// bytes the default pool holds beyond what is in use: they count as available for this call's scratch
static double pool_reserved_bytes() {
    int dev = 0;
    cudaMemPool_t pool;
    uint64_t reserved = 0, used = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetDefaultMemPool(&pool, dev) != cudaSuccess) return 0.0;
    if (cudaMemPoolGetAttribute(pool, cudaMemPoolAttrReservedMemCurrent, &reserved) != cudaSuccess) return 0.0;
    if (cudaMemPoolGetAttribute(pool, cudaMemPoolAttrUsedMemCurrent, &used) != cudaSuccess) return 0.0;
    return reserved > used ? (double)(reserved - used) : 0.0;
}
static int sm_count() {
    static thread_local int cached_dev = -1, cached = 132;   // H100 SXM
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (dev != cached_dev) {
        int v = 0;
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && v > 0) cached = v;
        cached_dev = dev;
    }
    return cached;
}

template <class C> struct MsmSession final : MsmSessionBase {
    using F = typename C::F;
    static constexpr int L = F::L;
    MsmGeom g;
    int kind = 0, levels_opt = -1, chunks_done = 0;
    size_t scalar_bytes = 32, n_seen = 0, max_chunk = 0;
    cudaStream_t st = 0;
    StreamArena arena;
    EventSet events;
    std::vector<cudaEvent_t> chunk_ev;   // 5 per chunk
    cudaEvent_t e_begin = nullptr, e_acc_done = nullptr, e_red = nullptr, e_end = nullptr;
    uint32_t *counts = nullptr, *offsets = nullptr, *sorted = nullptr, *block_totals = nullptr;
    uint32_t *buckets = nullptr, *extra = nullptr;
    size_t scan_blocks = 0;
    bool sliced = false;   // bucket slice of a larger MSM: entry counts are read back per chunk (they are ~1/slices of the bound)

    int coord_words() const override { return L; }

    int begin(size_t n_total, size_t max_chunk_, int kind_, cudaStream_t st_) override {
        st = st_;
        arena.st = st_;
        kind = kind_;
        max_chunk = max_chunk_;
        levels_opt = t_affine_levels;
        if (max_chunk >= ((size_t)1 << 31)) { set_last_error("chunk must be < 2^31 pairs"); return B200_ETOOLARGE; }
        const int scalar_bits = scalar_kind_bits(kind, C::SCALAR_BITS);
        scalar_bytes = scalar_kind_bytes(kind);
        int c = t_window_override ? t_window_override : msm_auto_window(std::max(n_total, max_chunk), scalar_bits);
        if (c > scalar_bits) c = scalar_bits;
        g = make_geom(c, scalar_bits, t_slice, t_slices);
        sliced = t_slices > 1;
        const size_t nb_total = g.total_buckets;
        const size_t max_entries = max_chunk * (size_t)g.W;
        if (max_entries >= ((size_t)1 << 31)) { set_last_error("chunk pairs * windows must be < 2^31"); return B200_ETOOLARGE; }
        scan_blocks = (nb_total + kScanBlock - 1) / kScanBlock;
        if (int rc = arena.alloc(&counts, nb_total * 4)) return rc;
        if (int rc = arena.alloc(&offsets, (nb_total + 1) * 4)) return rc;
        if (int rc = arena.alloc(&sorted, std::max<size_t>(max_entries, 1) * 4)) return rc;
        if (int rc = arena.alloc(&block_totals, std::max<size_t>(scan_blocks, 1) * 4)) return rc;
        if (int rc = arena.alloc(&buckets, nb_total * 4 * L * 4)) return rc;
        if (int rc = events.make(&e_begin)) return rc;
        if (int rc = events.make(&e_acc_done)) return rc;
        if (int rc = events.make(&e_red)) return rc;
        if (int rc = events.make(&e_end)) return rc;
        AB_CUDA(cudaEventRecord(e_begin, st));
        return 0;
    }

    int scan(const uint32_t *in, size_t n, uint32_t *out) {   // out[0..n] = exclusive prefix sums of in[0..n)
        const size_t blocks = (n + kScanBlock - 1) / kScanBlock;
        scan_block_totals_kernel<<<(unsigned)blocks, kScanThreads, 0, st>>>(in, n, block_totals);
        AB_LAUNCHED();
        scan_totals_kernel<<<1, kScanThreads, 0, st>>>(block_totals, blocks);
        AB_LAUNCHED();
        scan_apply_kernel<<<(unsigned)blocks, kScanThreads, 0, st>>>(in, n, block_totals, out);
        AB_LAUNCHED();
        return 0;
    }

    // XYZZ accumulation of `entries` bucket-ordered entries (bases gathered through `sorted_idx`, or direct affine points)
    // over the buckets [0, nbk) described by `offs`, written to `dst` (nbk buckets).
    int accumulate(const uint32_t *pts, const uint32_t *sorted_idx, const uint32_t *offs, size_t nbk, size_t entries, uint32_t *dst) {
        if (!entries) return 0;
        // balanced tasks: T entries per thread such that the grid is a whole number of waves (no tail), T <= 512
        const int blocks_per_sm = MsmAccLaunch<C>::occupancy(sorted_idx == nullptr);
        const double wave = (double)sm_count() * std::max(blocks_per_sm, 1) * 128.0;
        const double per_thread = (double)entries / wave;
        uint32_t T;
        if (per_thread <= 8.0) T = 8;
        else {
            const double waves = std::ceil(per_thread / 512.0);
            T = (uint32_t)std::ceil((double)entries / (waves * wave));
            T = std::min(512u, std::max(8u, T));
        }
        const uint32_t num_tasks = (uint32_t)((entries + T - 1) / T);
        uint32_t *head = nullptr, *tail = nullptr, *head_bucket = nullptr, *tail_bucket = nullptr;
        if (int rc = arena.alloc(&head, (size_t)num_tasks * 4 * L * 4)) return rc;
        if (int rc = arena.alloc(&tail, (size_t)num_tasks * 4 * L * 4)) return rc;
        if (int rc = arena.alloc(&head_bucket, (size_t)num_tasks * 4)) return rc;
        if (int rc = arena.alloc(&tail_bucket, (size_t)num_tasks * 4)) return rc;
        if (int rc = MsmAccLaunch<C>::accumulate(sorted_idx == nullptr, pts, sorted_idx, offs, (uint32_t)nbk, T, num_tasks, dst, head, tail, head_bucket,
                                                 tail_bucket, st))
            return rc;
        arena.release(head);
        arena.release(tail);
        arena.release(head_bucket);
        arena.release(tail_bucket);
        return 0;
    }

    // batched-affine levels + XYZZ accumulation of the buckets [b0, b1) (a group of whole windows) of the current chunk
    int reduce_group(const uint32_t *bas, size_t b0, size_t b1, size_t group_entries, int levels, uint32_t *target) {
        const size_t nbg = b1 - b0;
        const bool forced = levels_opt >= 0;
        size_t cur_entries = group_entries;   // upper bound on the entries of the current level
        const uint32_t *cur_src = sorted, *cur_offsets = offsets + b0;
        uint32_t *lvl_pts[2] = {nullptr, nullptr}, *lvl_off[2] = {nullptr, nullptr};
        int levels_done = 0;
        const double lanes_per_wave = (double)sm_count() * C::PAIR_MINB * 128;   // resident blocks of 128 threads
        for (int lv = 0; lv < levels; lv++) {
            // sum_b ceil(cnt_b / 2) <= min((entries + non-empty buckets) / 2, entries)
            const size_t out_cap = std::min((cur_entries + nbg) / 2 + 1, cur_entries);
            // one block-shared inversion (~590 modmuls) per 128 `batch` additions.  The grid is sized to a whole number of waves
            // of resident threads so that no SM idles through a partial last wave; in automatic mode a level that cannot give
            // every resident thread >= min_batch slots is left to the XYZZ kernel instead (measured: thin levels are slower).
            const double per_lane = (double)out_cap / lanes_per_wave;
            const double min_batch = (double)env_knobs().min_batch;
            if (!forced && per_lane < min_batch) break;
            const double waves = std::max(1.0, std::ceil(per_lane / 1024.0));
            uint32_t batch = (uint32_t)std::ceil((double)out_cap / (waves * lanes_per_wave));
            batch = std::min(1024u, std::max(forced ? 8u : (uint32_t)min_batch, batch));
            uint32_t *pts = nullptr, *off2 = nullptr;
            if (int rc = arena.alloc(&pts, out_cap * 2 * L * 4)) return rc;
            if (int rc = arena.alloc(&off2, (nbg + 1) * 4)) return rc;
            msm_halve_counts_kernel<<<(unsigned)((nbg + 255) / 256), 256, 0, st>>>(cur_offsets, (uint32_t)nbg, counts);
            AB_LAUNCHED();
            if (int rc = scan(counts, nbg, off2)) return rc;
            uint32_t *pairmap = nullptr;
            if (int rc = arena.alloc(&pairmap, out_cap * 4)) return rc;
            msm_pairmap_kernel<<<(unsigned)((out_cap + 1023) / 1024), 256, 0, st>>>(cur_offsets, off2, (uint32_t)nbg, pairmap);
            AB_LAUNCHED();
            if (int rc = MsmPairLaunch<C>::run(lv == 0, bas, cur_src, off2, pairmap, (uint32_t)nbg, batch, out_cap, pts, st)) return rc;
            arena.release(pairmap);
            // the level before the previous one is no longer read
            arena.release(lvl_pts[lv & 1]);
            arena.release(lvl_off[lv & 1]);
            lvl_pts[lv & 1] = pts;
            lvl_off[lv & 1] = off2;
            cur_src = pts;
            cur_offsets = off2;
            cur_entries = out_cap;
            levels_done++;
        }
        int rc;
        if (levels_done) rc = accumulate(cur_src, nullptr, cur_offsets, nbg, cur_entries, target + b0 * 4 * L);
        else rc = accumulate(bas, sorted, offsets + b0, nbg, group_entries, target + b0 * 4 * L);   // no level ran: gather through the sorted indices
        for (int q = 0; q < 2; q++) { arena.release(lvl_pts[q]); arena.release(lvl_off[q]); }
        return rc;
    }

    int add_chunk(const void *d_bases_v, const void *d_scalars, size_t nk, cudaEvent_t ready) override {
        if (nk > max_chunk) { set_last_error("chunk larger than announced at begin"); return B200_EINVAL; }
        const uint32_t *bas = (const uint32_t *)d_bases_v;
        const size_t nb_total = g.total_buckets;
        cudaEvent_t e[5];
        for (int i = 0; i < 5; i++) {
            if (int rc = events.make(&e[i])) return rc;
            chunk_ev.push_back(e[i]);
        }
        if (ready) AB_CUDA(cudaStreamWaitEvent(st, ready, 0));
        uint32_t *target = buckets;
        if (chunks_done > 0) {
            if (!extra)
                if (int rc = arena.alloc(&extra, nb_total * 4 * L * 4)) return rc;
            target = extra;
        }
        if (nb_total == 0) nk = 0;   // slice without buckets (a window with fewer buckets than slices goes whole to slice 0)
        AB_CUDA(cudaEventRecord(e[0], st));
        // bucket sort: digits (+ group counts) | bin plan | partition + bin sort.  Its scratch is released before the affine
        // levels, whose budget is taken from the free memory
        std::vector<size_t> upto((size_t)g.W + 1);   // entries of the chunk up to each window boundary
        for (int w = 0; w <= g.W; w++) upto[w] = nk * (size_t)w;
        uint32_t *digits = nullptr, *plan_mem = nullptr;
        uint2 *part = nullptr;
        MsmSortPlan plan;
        if (nk) {
            if (int rc = arena.alloc(&digits, nk * (size_t)g.W * 4)) return rc;
            if (int rc = arena.alloc(&plan_mem, MsmSortPlan::bytes(g.W))) return rc;
            plan.carve(plan_mem, g.W);
            AB_CUDA(cudaMemsetAsync(plan.gcount, 0, (size_t)g.W * kSortGroups * 4, st));
            if (int rc = MsmAccLaunch<C>::digits(d_scalars, kind, nk, g, digits, st)) return rc;
            if (int rc = msm_sort_count(digits, nk, g, plan, st)) return rc;
        }
        AB_CUDA(cudaEventRecord(e[1], st));
        if (nk) {
            if (int rc = msm_sort_plan(g, plan, offsets, st)) return rc;
            // a bucket slice receives only ~1/slices of the bound nk per window: its window bases are read back (the launch
            // geometry of the levels depends on them)
            if (sliced) {
                std::vector<uint32_t> h((size_t)g.W + 1, 0u);
                AB_CUDA(cudaMemcpyAsync(h.data(), plan.wbase, ((size_t)g.W + 1) * 4, cudaMemcpyDeviceToHost, st));
                AB_CUDA(cudaStreamSynchronize(st));
                for (int w = 0; w <= g.W; w++) upto[w] = h[w];
            }
        }
        const size_t entries = upto[g.W];
        AB_CUDA(cudaEventRecord(e[2], st));
        if (nk) {
            if (int rc = arena.alloc(&part, nk * sizeof(uint2))) return rc;
            if (int rc = msm_sort_scatter(digits, nk, g, plan, part, offsets, sorted, st)) return rc;
            arena.release(part);
            arena.release(plan_mem);
            arena.release(digits);
        }
        AB_CUDA(cudaEventRecord(e[3], st));
        AB_CUDA(cudaMemsetAsync(target, 0, nb_total * 4 * L * 4, st));
        if (nk && entries) {
            // batched-affine levels: automatic = keep halving while buckets still hold >= ~8 entries, at most 4 levels
            int levels = levels_opt;
            if (levels < 0) {
                levels = 0;
                if (C::AUTO_LEVELS)
                    for (double l = (double)nk / (double)(1u << (g.c - 1)); l >= env_knobs().level_min_load && levels < std::min(env_knobs().level_cap, C::LEVEL_CAP); l *= 0.5) levels++;
                // the first level must be able to give every resident thread a batch of >= min_batch additions
                if ((double)entries * 0.5 / ((double)sm_count() * C::PAIR_MINB * 128.0) < (double)env_knobs().min_batch) levels = 0;
            }
            if (levels == 0) {
                if (int rc = accumulate(bas, sorted, offsets, nb_total, entries, target)) return rc;
            } else {
                // window groups: the level arrays of one group (level 1: entries/2 affine points, level 2: half of that, two
                // levels alive at a time) must fit the scratch budget; groups are whole windows, balanced in size
                const double ew = (double)entries / g.W;   // entries per window
                const double per_window = (ew * 0.5 + (double)g.nb * 0.5) * 2 * L * 4 * 1.5 + ew * 0.5 * 4;
                double budget = env_knobs().level_budget_bytes;
                size_t free_b = 0, total_b = 0;
                if (cudaMemGetInfo(&free_b, &total_b) == cudaSuccess) budget = std::min(budget, 0.6 * (double)free_b + pool_reserved_bytes());
                int gw = (int)std::floor(budget / per_window);
                // ... and a group must give every resident thread a batch of >= min_batch additions at level 1
                const int gw_min = (int)std::ceil((double)env_knobs().min_batch * (double)sm_count() * C::PAIR_MINB * 128.0 / std::max(1.0, ew * 0.5));
                gw = std::max(std::max(1, gw_min), std::min(g.W, gw));
                gw = std::min(g.W, gw);
                const int ngroups = (g.W + gw - 1) / gw;
                gw = (g.W + ngroups - 1) / ngroups;
                for (int w0 = 0; w0 < g.W; w0 += gw) {
                    const int w1 = std::min(g.W, w0 + gw);
                    const size_t b0 = (size_t)w0 * g.nb, b1 = (w1 == g.W) ? nb_total : (size_t)w1 * g.nb;
                    if (int rc = reduce_group(bas, b0, b1, upto[w1] - upto[w0], levels, target)) return rc;
                }
            }
        }
        if (chunks_done > 0) {
            if (int rc = MsmAccLaunch<C>::merge(buckets, extra, (uint32_t)nb_total, st)) return rc;
        }
        AB_CUDA(cudaEventRecord(e[4], st));
        chunks_done++;
        n_seen += nk;
        return 0;
    }

    int finish(void *d_out_v) override {
        uint32_t *d_out = (uint32_t *)d_out_v;
        const size_t nb_total = g.total_buckets;
        if (chunks_done == 0) AB_CUDA(cudaMemsetAsync(buckets, 0, nb_total * 4 * L * 4, st));
        AB_CUDA(cudaEventRecord(e_acc_done, st));
        // reduction geometry: chunk of m = 2^log_m buckets per thread
        // (each thread pays ~300 multiplications for its chunk-offset product on top of 28 per bucket: longer chunks amortise it, as long as
        // W * nb / m threads still fill the machine a few times over)
        int log_m = env_knobs().reduce_log_m;
        while (!env_knobs().reduce_log_m_forced && log_m > 5 && ((size_t)g.W * g.nb >> log_m) < (size_t)sm_count() * 512) log_m--;
        while (log_m > 0 && (g.nb >> log_m) < 64) log_m--;
        const uint32_t max_nb = std::max(g.nb, g.nb_top);
        const uint32_t chunks = (max_nb + (1u << log_m) - 1) >> log_m;
        uint32_t *partials = nullptr, *partials2 = nullptr, *window_sums = nullptr;
        if (int rc = arena.alloc(&partials, (size_t)g.W * chunks * 4 * L * 4)) return rc;
        if (int rc = arena.alloc(&partials2, (size_t)g.W * 32 * 4 * L * 4)) return rc;
        if (int rc = arena.alloc(&window_sums, (size_t)g.W * 4 * L * 4)) return rc;
        if (nb_total == 0) AB_CUDA(cudaMemsetAsync(window_sums, 0, (size_t)g.W * 4 * L * 4, st));   // empty slice: the identity
        else if (int rc = MsmRedLaunch<C>::reduce(buckets, g, log_m, chunks, partials, partials2, window_sums, st)) return rc;
        AB_CUDA(cudaEventRecord(e_red, st));
        if (int rc = MsmRedLaunch<C>::combine(window_sums, g.W, g.c, d_out, st)) return rc;
        AB_CUDA(cudaEventRecord(e_end, st));
        return 0;
    }

    int collect_timings() override {
        for (int i = 0; i < 7; i++) t_last.ms[i] = 0.f;
        for (size_t k = 0; k + 4 < chunk_ev.size(); k += 5)
            for (int i = 0; i < 4; i++) {
                float ms = 0.f;
                AB_CUDA(cudaEventElapsedTime(&ms, chunk_ev[k + i], chunk_ev[k + i + 1]));
                t_last.ms[i] += ms;  // digits+hist, scan, scatter, accumulate(+fixups, merge)
            }
        AB_CUDA(cudaEventElapsedTime(&t_last.ms[4], e_acc_done, e_red));
        AB_CUDA(cudaEventElapsedTime(&t_last.ms[5], e_red, e_end));
        AB_CUDA(cudaEventElapsedTime(&t_last.ms[6], e_begin, e_end));  // includes waiting for transfers on the host paths
        t_last.c = g.c;
        t_last.W = g.W;
        t_last.bucket_adds = (unsigned long long)n_seen * g.W;  // upper bound: zero digits are skipped
        return 0;
    }
};

MsmSessionBase *msm_session_create(int curve) {
    switch (curve) {
        case B200_CURVE_BLS12_381: return new MsmSession<CurveBls>();
        case B200_CURVE_BN254: return new MsmSession<CurveBn>();
        case B200_CURVE_BLS12_381_G2: return new MsmSession<CurveBlsG2>();
    }
    return nullptr;
}
const CurveInfo *curve_info(int curve) {
    static const CurveInfo bls = {CurveBls::F::L, CurveBls::SCALAR_BITS, B200_FIELD_BLS12_381_FR},
                           bn = {CurveBn::F::L, CurveBn::SCALAR_BITS, B200_FIELD_BN254_FR},
                           g2 = {CurveBlsG2::F::L, CurveBlsG2::SCALAR_BITS, B200_FIELD_BLS12_381_FR};
    switch (curve) {
        case B200_CURVE_BLS12_381: return &bls;
        case B200_CURVE_BN254: return &bn;
        case B200_CURVE_BLS12_381_G2: return &g2;
    }
    return nullptr;
}
const FieldInfo *field_info(int field) {
    static const FieldInfo bls = {BlsFr::TWO_ADICITY, 1}, bn = {BnFr::TWO_ADICITY, 3};
    switch (field) {
        case B200_FIELD_BLS12_381_FR: return &bls;
        case B200_FIELD_BN254_FR: return &bn;
    }
    return nullptr;
}
static uint32_t curve_one_limb(int curve, int i) {   // Montgomery ONE of the coordinate field, 32-bit word i
    switch (curve) {
        case B200_CURVE_BLS12_381: return BlsFq::ONE(i);
        case B200_CURVE_BN254: return BnFq::ONE(i);
        default: return i < 12 ? BlsFq::ONE(i) : 0u;   // Fq2 one = (1, 0)
    }
}
// Projective::zero() = (1,1,0) (group.rs:142-158) as 3 coordinates of L words, written as u64 limbs
void msm_write_zero(int curve, uint64_t *out_xyz) {
    const int L = curve_info(curve)->coord_words;
    for (int i = 0; i < 3 * L / 2; i++) out_xyz[i] = 0;
    for (int k = 0; k < 2; k++)
        for (int i = 0; i < L; i++) out_xyz[(k * L + i) / 2] |= (uint64_t)curve_one_limb(curve, i) << (32 * ((k * L + i) & 1));
}

// One MSM over K chunks of device-resident (or in-flight: `ready` events) inputs.  Each chunk is digit-sorted and accumulated
// as soon as its event fires, so the host paths overlap the PCIe transfer of chunk k+1 with the arithmetic of chunk k; the
// bucket reduction and window combine run once at the end.
int msm_dispatch(int curve, int kind, const void *d_bases, const void *d_scalars, size_t n, uint64_t *out_xyz_host, cudaStream_t st, int K,
                 const size_t *chunk_off, const cudaEvent_t *ready) {
    if (int rc = check_scalar_kind(kind)) return rc;
    if (!out_xyz_host || (n && (!d_bases || !d_scalars))) { set_last_error("null pointer"); return B200_EINVAL; }
    const CurveInfo *ci = curve_info(curve);
    if (!ci) { set_last_error("unknown curve id"); return B200_EINVAL; }
    if (n == 0) { msm_write_zero(curve, out_xyz_host); return 0; }
    if (n >= ((size_t)1 << 31)) { set_last_error("n must be < 2^31"); return B200_ETOOLARGE; }
    // device-resident inputs too large for one 31-bit entry index space (n * windows >= 2^31): split into equal chunks
    std::vector<size_t> auto_off;
    const int force = env_knobs().force_chunks;   // test hook: exercise the chunked device path at small n
    if (K <= 1) {
        int kk = 1;
        if (n > ((size_t)1 << 27)) kk = (int)((n + ((size_t)1 << 27) - 1) >> 27);
        else if (force > 1 && n >= 64) kk = force;
        for (int k = 0; k <= kk; k++) auto_off.push_back(n * (size_t)k / kk);
        K = kk;
        chunk_off = auto_off.data();
        ready = nullptr;
    }
    size_t max_chunk = 0;
    for (int k = 0; k < K; k++) max_chunk = std::max(max_chunk, chunk_off[k + 1] - chunk_off[k]);
    std::unique_ptr<MsmSessionBase> s(msm_session_create(curve));
    const size_t sb = scalar_kind_bytes(kind);
    int rc = s->begin(n, max_chunk, kind, st);
    for (int k = 0; k < K && !rc; k++)
        rc = s->add_chunk((const char *)d_bases + chunk_off[k] * (size_t)(2 * ci->coord_words * 4), (const char *)d_scalars + chunk_off[k] * sb,
                          chunk_off[k + 1] - chunk_off[k], ready ? ready[k] : nullptr);
    if (rc) { cudaStreamSynchronize(st); return rc; }   // nothing of this call is in flight when it returns
    return msm_session_result(*s, out_xyz_host, st);   // ~MsmSession frees the scratch and the events
}

int msm_session_result(MsmSessionBase &s, uint64_t *out_xyz, cudaStream_t st) {
    const size_t bytes = (size_t)3 * s.coord_words() * 4;
    void *d_out = nullptr;
    int rc = 0;
    cudaError_t e = cudaMallocAsync(&d_out, bytes, st);
    if (e != cudaSuccess) rc = cuda_fail(e, "cudaMallocAsync", __FILE__, __LINE__);
    if (!rc) rc = s.finish(d_out);
    if (!rc) {
        e = cudaMemcpyAsync(out_xyz, d_out, bytes, cudaMemcpyDeviceToHost, st);
        if (e != cudaSuccess) rc = cuda_fail(e, "cudaMemcpyAsync D2H", __FILE__, __LINE__);
    }
    if (d_out) cudaFreeAsync(d_out, st);
    e = cudaStreamSynchronize(st);   // also on the error paths: nothing of the session's work is in flight when it returns
    if (!rc && e != cudaSuccess) rc = cuda_fail(e, "cudaStreamSynchronize", __FILE__, __LINE__);
    if (!rc) rc = s.collect_timings();
    return rc;
}

int msm_last_timings(float *ms7, int *c, int *windows, unsigned long long *bucket_adds) {
    if (ms7) for (int i = 0; i < 7; i++) ms7[i] = t_last.ms[i];
    if (c) *c = t_last.c;
    if (windows) *windows = t_last.W;
    if (bucket_adds) *bucket_adds = t_last.bucket_adds;
    return 0;
}

int g1_sum(int curve, const void *d_pts, size_t k, void *d_out, bool to_affine, cudaStream_t st) {
    const uint32_t *in = (const uint32_t *)d_pts;
    uint32_t *out = (uint32_t *)d_out;
    switch (curve) {
        case B200_CURVE_BLS12_381: return MsmRedLaunch<CurveBls>::sum_or_affine(to_affine, in, k, out, st);
        case B200_CURVE_BN254: return MsmRedLaunch<CurveBn>::sum_or_affine(to_affine, in, k, out, st);
        case B200_CURVE_BLS12_381_G2: return MsmRedLaunch<CurveBlsG2>::sum_or_affine(to_affine, in, k, out, st);
    }
    set_last_error("unknown curve id");
    return B200_EINVAL;
}

}  // namespace ab200

