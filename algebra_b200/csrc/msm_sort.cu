// msm_sort.cu — bucket sort of one chunk's MSM entries: from the window-major digit array (msm_digits_kernel) to `offsets`
// (exclusive prefix of the bucket sizes, bucket id = w * nb + rel) and `sorted` (index | sign << 31 in bucket order).
// No per-entry global atomic and no scattered 4-byte store into a multi-GB array:
//   count      per window, a shared-memory histogram of the digits over G <= 8192 groups of 2^gs buckets, one global add per
//              (block, group)
//   plan       per window, one block: scan of the group counts; the groups are joined into bins (sort_bin_of / sort_bin_height,
//              msm_common.cuh) of at most kSortCap entries and kSortSpan buckets; window bases for the chunk
//   partition  per window: each block counts its tile per bin in shared memory, reserves one run per bin with one global add,
//              sorts the tile by bin in shared memory and writes (rel, index | sign) run by run, coalesced
//   bins       per window, one block per bin: histogram of the bin's buckets, scan -> offsets, placement into a shared copy
//              of the bin, coalesced copy to `sorted`.  A bin above kSortCap (only when one group alone holds more than
//              kSortCap / 2 entries: skewed scalars) places its entries straight into `sorted` instead
// The order of the entries inside a bucket depends on the scheduling of the blocks; the group element does not.
#include "msm_common.cuh"

namespace ab200 {

static constexpr int kCountThreads = 1024, kPlanThreads = 1024, kPartThreads = 1024, kBinThreads = 512;
static constexpr uint32_t kCountTile = 1u << 18, kPartTile = 1u << 14;

__device__ __forceinline__ uint32_t window_buckets(const MsmGeom &g, int w) { return w == g.W - 1 ? g.nb_top : g.nb; }

// exclusive scan over the block (blockDim.x a multiple of 32, <= 1024); *total = sum over the block
__device__ __forceinline__ uint32_t sort_block_scan(uint32_t v, uint32_t *total) {
    __shared__ uint32_t warp_sums[32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[wid] = x;
    __syncthreads();
    if (wid == 0) {
        uint32_t ws = lane < nw ? warp_sums[lane] : 0;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, ws, o);
            if (lane >= o) ws += y;
        }
        warp_sums[lane] = ws;
    }
    __syncthreads();
    const uint32_t r = (wid ? warp_sums[wid - 1] : 0) + x - v;
    *total = warp_sums[nw - 1];
    __syncthreads();   // warp_sums may be reused by the next call
    return r;
}

// grid (tiles, W)
__global__ void __launch_bounds__(kCountThreads) msm_sort_count_kernel(const uint32_t *__restrict__ digits, uint32_t nk, MsmGeom g,
                                                                       uint32_t *__restrict__ gcount) {
    __shared__ uint32_t h[kSortGroups];
    const int w = blockIdx.y;
    const MsmSortWin s = sort_window(window_buckets(g, w));
    for (uint32_t j = threadIdx.x; j < s.G; j += blockDim.x) h[j] = 0;
    __syncthreads();
    const uint32_t *d = digits + (size_t)w * nk;
    const uint32_t lo = blockIdx.x * kCountTile, hi = min(nk, lo + kCountTile);
#pragma unroll 4
    for (uint32_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
        const uint32_t v = __ldg(d + i);
        if (v != kNoDigit) atomicAdd(&h[(v & 0x7fffffffu) >> s.gs], 1u);
    }
    __syncthreads();
    for (uint32_t j = threadIdx.x; j < s.G; j += blockDim.x)
        if (h[j]) atomicAdd(&gcount[(size_t)w * kSortGroups + j], h[j]);
}

// grid W, one block per window
__global__ void __launch_bounds__(kPlanThreads) msm_sort_plan_kernel(MsmGeom g, MsmSortPlan p, uint32_t *__restrict__ offsets_end) {
    constexpr uint32_t PER = kSortGroups / kPlanThreads;
    __shared__ uint32_t s_max;
    const int w = blockIdx.x;
    const MsmSortWin s = sort_window(window_buckets(g, w));
    const uint32_t *cnt = p.gcount + (size_t)w * kSortGroups;
    // entries of the earlier windows (their unused groups are zero)
    uint32_t before = 0;
    for (size_t j = threadIdx.x; j < (size_t)w * kSortGroups; j += blockDim.x) before += p.gcount[j];
    uint32_t base;
    sort_block_scan(before, &base);
    if (threadIdx.x == 0) s_max = 0;
    uint32_t c[PER], sum = 0, mx = 0;
    const uint32_t g0 = threadIdx.x * PER;
#pragma unroll
    for (int q = 0; q < (int)PER; q++) {
        c[q] = g0 + q < s.G ? cnt[g0 + q] : 0;
        sum += c[q];
        mx = max(mx, c[q]);
    }
    __syncthreads();
    atomicMax(&s_max, mx);
    uint32_t total;
    uint32_t start = sort_block_scan(sum, &total);   // also orders the atomicMax before the read of s_max
    const uint32_t h = sort_bin_height(total, s_max, s.G, s.gpb);
    uint32_t *bstart = p.bstart + (size_t)w * (kSortBins + 1), *bgroup = p.bgroup + (size_t)w * (kSortBins + 1);
    uint32_t *bcur = p.bcur + (size_t)w * kSortBins;
    uint16_t *gbin = p.gbin + (size_t)w * kSortGroups;
    // group gi opens the bins (bin of gi-1, bin of gi]: empty bins between two groups start where the next group starts
    uint32_t prev = (g0 == 0 || g0 >= s.G) ? 0xffffffffu : sort_bin_of(start - cnt[g0 - 1], g0 - 1, h, s.gpb);
#pragma unroll
    for (int q = 0; q < (int)PER; q++) {
        const uint32_t gi = g0 + q;
        if (gi < s.G) {
            const uint32_t k = sort_bin_of(start, gi, h, s.gpb);
            for (uint32_t kk = prev + 1; kk <= k; kk++) {
                bstart[kk] = start;
                bgroup[kk] = gi;
                bcur[kk] = start;
            }
            gbin[gi] = (uint16_t)k;
            if (gi == s.G - 1) {
                bstart[k + 1] = total;
                bgroup[k + 1] = s.G;
                p.nbins[w] = k + 1;
            }
            prev = k;
        }
        start += c[q];
    }
    if (threadIdx.x == 0) {
        if (s.G == 0) {
            bstart[0] = 0;
            bgroup[0] = 0;
            p.nbins[w] = 0;
        }
        p.wbase[w] = base;
        if (w == g.W - 1) {
            p.wbase[g.W] = base + total;
            *offsets_end = base + total;
        }
    }
}

// one window; grid = tiles of kPartTile entries.  The tile is sorted by bin in shared memory and every run is written in one
// coalesced burst, so the runs of the blocks in flight fill whole sectors while they are in L2.  Dynamic shared memory:
// 2 x nbins_max counters + kPartTile staged entries
__global__ void __launch_bounds__(kPartThreads) msm_sort_partition_kernel(const uint32_t *__restrict__ digits, uint32_t nk, uint32_t gs,
                                                                          const uint16_t *__restrict__ gbin, const uint32_t *__restrict__ nbins_p,
                                                                          uint32_t nbins_max, uint32_t *__restrict__ bcur, uint2 *__restrict__ part) {
    extern __shared__ uint2 sm2[];
    uint2 *stage = sm2;
    uint32_t *loc = (uint32_t *)(sm2 + kPartTile), *gpos = loc + nbins_max;
    const uint32_t nbins = *nbins_p;
    for (uint32_t j = threadIdx.x; j < nbins; j += blockDim.x) loc[j] = 0;
    __syncthreads();
    const uint32_t lo = blockIdx.x * kPartTile, hi = min(nk, lo + kPartTile);
#pragma unroll 4
    for (uint32_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {
        const uint32_t v = __ldg(digits + i);
        if (v != kNoDigit) atomicAdd(&loc[__ldg(gbin + ((v & 0x7fffffffu) >> gs))], 1u);
    }
    __syncthreads();
    // local run starts (exclusive scan) and one global reservation per (block, bin): gpos = global start - local start
    const uint32_t per = (nbins + blockDim.x - 1) / blockDim.x, j0 = min(nbins, threadIdx.x * per), j1 = min(nbins, j0 + per);
    uint32_t sum = 0;
    for (uint32_t j = j0; j < j1; j++) sum += loc[j];
    uint32_t staged;
    uint32_t ex = sort_block_scan(sum, &staged);
    for (uint32_t j = j0; j < j1; j++) {
        const uint32_t c = loc[j];
        loc[j] = ex;
        gpos[j] = c ? atomicAdd(&bcur[j], c) - ex : 0u;
        ex += c;
    }
    __syncthreads();
#pragma unroll 4
    for (uint32_t i = lo + threadIdx.x; i < hi; i += blockDim.x) {   // the tile is re-read from L2
        const uint32_t v = __ldg(digits + i);
        if (v != kNoDigit) {
            const uint32_t rel = v & 0x7fffffffu;
            stage[atomicAdd(&loc[__ldg(gbin + (rel >> gs))], 1u)] = make_uint2(rel, i | (v & 0x80000000u));
        }
    }
    __syncthreads();
    for (uint32_t j = threadIdx.x; j < staged; j += blockDim.x) {
        const uint2 e = stage[j];
        part[gpos[__ldg(gbin + (e.x >> gs))] + j] = e;
    }
}

// one window; grid = upper bound on its bins (sort_max_bins), one block per bin.  Dynamic shared memory:
// kSortSpan bucket counters + kSortCap staged entries
__global__ void __launch_bounds__(kBinThreads, 2) msm_sort_bins_kernel(const uint2 *__restrict__ part, const uint32_t *__restrict__ bstart,
                                                                        const uint32_t *__restrict__ bgroup, const uint32_t *__restrict__ nbins_p,
                                                                        const uint32_t *__restrict__ wbase_p, uint32_t gs, uint32_t nbw, uint32_t bucket0,
                                                                        uint32_t *__restrict__ offsets, uint32_t *__restrict__ sorted) {
    extern __shared__ uint32_t sm[];
    uint32_t *hist = sm, *stage = sm + kSortSpan;
    const uint32_t k = blockIdx.x;
    if (k >= *nbins_p) return;
    const uint32_t e0 = bstart[k], e1 = bstart[k + 1];
    const uint32_t b_lo = bgroup[k] << gs, b_hi = min(bgroup[k + 1] << gs, nbw), span = b_hi - b_lo;   // span <= kSortSpan
    const uint32_t out = *wbase_p + e0, n = e1 - e0;
    for (uint32_t j = threadIdx.x; j < span; j += blockDim.x) hist[j] = 0;
    __syncthreads();
    for (uint32_t i = e0 + threadIdx.x; i < e1; i += blockDim.x) atomicAdd(&hist[part[i].x - b_lo], 1u);
    __syncthreads();
    // exclusive scan of hist[0, span): kSortSpan / kBinThreads consecutive counters per thread
    constexpr uint32_t PER = kSortSpan / kBinThreads;
    uint32_t v[PER], sum = 0;
    const uint32_t j0 = threadIdx.x * PER;
#pragma unroll
    for (int q = 0; q < (int)PER; q++) {
        v[q] = j0 + q < span ? hist[j0 + q] : 0;
        sum += v[q];
    }
    uint32_t total;
    uint32_t ex = sort_block_scan(sum, &total);
#pragma unroll
    for (int q = 0; q < (int)PER; q++) {
        if (j0 + q < span) {
            hist[j0 + q] = ex;
            offsets[bucket0 + b_lo + j0 + q] = out + ex;
        }
        ex += v[q];
    }
    __syncthreads();
    if (n <= kSortCap) {
        for (uint32_t i = e0 + threadIdx.x; i < e1; i += blockDim.x) {
            const uint2 e = part[i];
            stage[atomicAdd(&hist[e.x - b_lo], 1u)] = e.y;
        }
        __syncthreads();
        for (uint32_t j = threadIdx.x; j < n; j += blockDim.x) sorted[out + j] = stage[j];
    } else {
        for (uint32_t i = e0 + threadIdx.x; i < e1; i += blockDim.x) {
            const uint2 e = part[i];
            sorted[out + atomicAdd(&hist[e.x - b_lo], 1u)] = e.y;
        }
    }
}

int msm_sort_count(const uint32_t *digits, size_t nk, const MsmGeom &g, const MsmSortPlan &plan, cudaStream_t st) {
    const dim3 grid((unsigned)((nk + kCountTile - 1) / kCountTile), (unsigned)g.W);
    msm_sort_count_kernel<<<grid, kCountThreads, 0, st>>>(digits, (uint32_t)nk, g, plan.gcount);
    AB_LAUNCHED();
    return 0;
}

int msm_sort_plan(const MsmGeom &g, const MsmSortPlan &plan, uint32_t *offsets, cudaStream_t st) {
    msm_sort_plan_kernel<<<(unsigned)g.W, kPlanThreads, 0, st>>>(g, plan, offsets + g.total_buckets);
    AB_LAUNCHED();
    return 0;
}

int msm_sort_scatter(const uint32_t *digits, size_t nk, const MsmGeom &g, const MsmSortPlan &plan, uint2 *part, uint32_t *offsets, uint32_t *sorted,
                     cudaStream_t st) {
    const size_t smem = (size_t)(kSortSpan + kSortCap) * 4;
    AB_CUDA(cudaFuncSetAttribute(msm_sort_bins_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    AB_CUDA(cudaFuncSetAttribute(msm_sort_partition_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(kPartTile * 8 + kSortBins * 8)));
    for (int w = 0; w < g.W; w++) {
        const uint32_t nbw = w == g.W - 1 ? g.nb_top : g.nb;
        if (!nbw) continue;
        const MsmSortWin s = sort_window(nbw);
        const uint32_t max_bins = sort_max_bins(nk, nbw);
        msm_sort_partition_kernel<<<(unsigned)((nk + kPartTile - 1) / kPartTile), kPartThreads, (size_t)kPartTile * 8 + (size_t)max_bins * 8, st>>>(
            digits + (size_t)w * nk, (uint32_t)nk, s.gs, plan.gbin + (size_t)w * kSortGroups, plan.nbins + w, max_bins, plan.bcur + (size_t)w * kSortBins, part);
        AB_LAUNCHED();
        msm_sort_bins_kernel<<<max_bins, kBinThreads, smem, st>>>(part, plan.bstart + (size_t)w * (kSortBins + 1),
                                                                                plan.bgroup + (size_t)w * (kSortBins + 1), plan.nbins + w, plan.wbase + w, s.gs,
                                                                                nbw, (uint32_t)w * g.nb, offsets, sorted);
        AB_LAUNCHED();
    }
    return 0;
}

}  // namespace ab200
