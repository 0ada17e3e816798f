// capi.cu — the extern "C" boundary declared in include/algebra_b200.h.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>
#include "common.cuh"

namespace ab200 {
int ntt_dispatch(int field, void *d_data, uint32_t log_n, int inverse, const uint64_t *coset, cudaStream_t st);
int ntt_clear_cache();
int point_ntt_check(int curve, const void *points, uint32_t log_n);
int point_ntt_coord_words(int curve);
int point_ntt_dispatch(int curve, void *d_points, uint32_t log_n, int inverse, const uint64_t *coset, cudaStream_t st);
struct MsmSessionBase {
    virtual ~MsmSessionBase() {}
    virtual int begin(size_t n_total, size_t max_chunk, int kind, cudaStream_t st) = 0;
    virtual int add_chunk(const void *d_bases, const void *d_scalars, size_t nk, cudaEvent_t ready) = 0;
    virtual int finish(void *d_out) = 0;
    virtual int collect_timings() = 0;
    virtual int coord_words() const = 0;
};
MsmSessionBase *msm_session_create(int curve);
int msm_coord_words(int curve);
void msm_write_zero(int curve, uint64_t *out_xyz);
int msm_dispatch(int curve, int kind, const void *d_bases, const void *d_scalars, size_t n, uint64_t *out_xyz_host, cudaStream_t st, int K,
                 const size_t *chunk_off, const cudaEvent_t *ready);
size_t scalar_kind_bytes(int kind);
int msm_set_window(int c);
int msm_set_affine_levels(int levels);
int msm_get_window();
int msm_get_affine_levels();
int msm_set_bucket_slice(int slice, int slices);
void msm_get_bucket_slice(int *slice, int *slices);
int msm_auto_window(size_t n, int scalar_bits);
int msm_last_timings(float *ms7, int *c, int *windows, unsigned long long *bucket_adds);
int g1_sum_dispatch(int curve, const uint64_t *pts_host, size_t k, uint64_t *out_host, bool to_affine);
int fp_op_dispatch(int field, int op, const void *a, const void *b, void *out, size_t n, int reps, cudaStream_t st);
int ec_op_dispatch(int curve, int op, const void *a, const void *b, void *out, size_t n, cudaStream_t st);
int gen_bases_dispatch(int curve, uint64_t seed, size_t n, void *d_bases, void *d_b, cudaStream_t st);
int gen_scalars_dispatch(int field, uint64_t seed, size_t n, void *d_scalars, cudaStream_t st);
int batch_mul_dispatch(int curve, const uint64_t *base_xy, const void *d_scalars, size_t n, void *d_out, cudaStream_t st);
int normalize_batch_dispatch(int curve, const void *d_xyz, size_t n, void *d_out, cudaStream_t st);

// ------------------------------------------------------------------------------------------------
// Host-buffer plumbing: per-device contexts (compute stream, copy stream, pinned staging ring), leased per call so that
// concurrent callers and the per-device worker threads of the multi-GPU entry points never share one.
// ------------------------------------------------------------------------------------------------
static constexpr size_t kRingSlot = (size_t)16 << 20;   // bytes per pinned staging slot
static constexpr int kCopyThreads = 8, kRingSlots = 2 * kCopyThreads;   // several threads: one memcpy thread cannot fill the ring as fast as PCIe drains it

struct DeviceCtx {
    int dev = 0;
    cudaStream_t st = nullptr, copy_st = nullptr;
    void *ring[kRingSlots] = {};
    cudaEvent_t ring_ev[kRingSlots] = {};
    bool ring_ready = false;
    int init(int d) {
        dev = d;
        AB_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
        AB_CUDA(cudaStreamCreateWithFlags(&copy_st, cudaStreamNonBlocking));
        return 0;
    }
    int init_ring() {   // only callers with pageable buffers pay for the pinned ring
        if (ring_ready) return 0;
        for (int i = 0; i < kRingSlots; i++) {
            AB_CUDA(cudaHostAlloc(&ring[i], kRingSlot, cudaHostAllocDefault));
            AB_CUDA(cudaEventCreateWithFlags(&ring_ev[i], cudaEventDisableTiming));
        }
        ring_ready = true;
        return 0;
    }
};
static std::mutex g_ctx_mutex;
static std::vector<DeviceCtx *> g_free_ctx[64];

struct CtxLease {
    DeviceCtx *c = nullptr;
    int acquire(int dev) {
        if (dev < 0 || dev >= 64) { set_last_error("device index out of range"); return B200_EINVAL; }
        {
            std::lock_guard<std::mutex> lk(g_ctx_mutex);
            if (!g_free_ctx[dev].empty()) { c = g_free_ctx[dev].back(); g_free_ctx[dev].pop_back(); return 0; }
        }
        std::unique_ptr<DeviceCtx> n(new DeviceCtx());
        if (int rc = n->init(dev)) return rc;
        c = n.release();
        return 0;
    }
    ~CtxLease() {
        if (!c) return;
        std::lock_guard<std::mutex> lk(g_ctx_mutex);
        g_free_ctx[c->dev].push_back(c);
    }
};

static bool is_pageable(const void *p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return true; }
    return a.type == cudaMemoryTypeUnregistered;
}

// dst (device) <- src (host), enqueued on c.copy_st.  Pinned / registered sources: one asynchronous copy.  Pageable sources:
// kCopyThreads host threads memcpy alternating slices into their two pinned ring slots and enqueue the DMA of each slice, so
// host memcpy and PCIe transfer overlap; returns when every slice has been ENQUEUED (the ring keeps the data alive).
static int h2d(DeviceCtx &c, void *dst, const void *src, size_t bytes) {
    if (!bytes) return 0;
    if (!is_pageable(src)) {
        AB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, c.copy_st));
        return 0;
    }
    if (int rc = c.init_ring()) return rc;
    const size_t slices = (bytes + kRingSlot - 1) / kRingSlot;
    const int T = (int)std::min<size_t>(kCopyThreads, slices);
    std::vector<cudaError_t> err((size_t)T, cudaSuccess);
    auto worker = [&](int t) {
        cudaError_t e = cudaSetDevice(c.dev);
        for (size_t s = (size_t)t, it = 0; s < slices && e == cudaSuccess; s += (size_t)T, it++) {
            const int slot = 2 * t + (int)(it & 1);
            const size_t off = s * kRingSlot, len = std::min(kRingSlot, bytes - off);
            e = cudaEventSynchronize(c.ring_ev[slot]);   // the previous DMA out of this slot has finished
            if (e != cudaSuccess) break;
            memcpy(c.ring[slot], (const char *)src + off, len);
            e = cudaMemcpyAsync((char *)dst + off, c.ring[slot], len, cudaMemcpyHostToDevice, c.copy_st);
            if (e == cudaSuccess) e = cudaEventRecord(c.ring_ev[slot], c.copy_st);
        }
        err[(size_t)t] = e;
    };
    std::vector<std::thread> th;
    for (int t = 1; t < T; t++) th.emplace_back(worker, t);
    worker(0);
    for (auto &x : th) x.join();
    for (cudaError_t e : err)
        if (e != cudaSuccess) return cuda_fail(e, "staged host-to-device copy", __FILE__, __LINE__);
    return 0;
}

// chunk boundaries of the host path in 16ths of n.  Growing chunks: only the first, small transfer is exposed and every later
// one is shorter than the arithmetic of the chunk before it; few chunks, because small chunks run the accumulation less
// efficiently (short bucket runs) and each extra chunk costs a bucket-merge pass.  B200_MSM_CHUNKS="2,8,16" overrides (read once).
struct ChunkPlan {
    int K = 3;
    int bounds[9] = {0, 2, 7, 16, 0, 0, 0, 0, 0};
    ChunkPlan() {
        if (const char *e = getenv("B200_MSM_CHUNKS")) {
            int b[9] = {0}, k = 0, v = 0;
            const char *q = e;
            while (*q && k < 8) {
                v = atoi(q);
                if (v <= b[k] || v > 16) break;
                b[++k] = v;
                while (*q && *q != ',') q++;
                if (*q == ',') q++;
            }
            if (k >= 1 && b[k] == 16) { K = k; for (int i = 0; i <= k; i++) bounds[i] = b[i]; }
        }
    }
};
static const ChunkPlan &chunk_plan() {
    static const ChunkPlan p;
    return p;
}

// The whole host-buffer MSM on the CURRENT device: allocate, pipeline (H2D chunk k+1 | sort + accumulate chunk k), reduce,
// D2H.  `d_bases_resident` != null: the bases already live on this device and only the scalars travel.
static int host_msm(int curve, int kind, const void *bases, const void *d_bases_resident, const void *scalars, size_t n, uint64_t *out_xyz) {
    const int L = msm_coord_words(curve);
    if (n == 0) { msm_write_zero(curve, out_xyz); return 0; }
    int dev = 0;
    AB_CUDA(cudaGetDevice(&dev));
    CtxLease lease;
    if (int rc = lease.acquire(dev)) return rc;
    DeviceCtx &c = *lease.c;
    const size_t sb = scalar_kind_bytes(kind), pb = (size_t)2 * L * 4;
    const ChunkPlan &plan = chunk_plan();
    const int K = n >= ((size_t)1 << 22) ? plan.K : 1;
    size_t off[9];
    for (int k = 0; k <= K; k++) off[k] = K == 1 ? (size_t)k * n : n / 16 * (size_t)plan.bounds[k];
    off[K] = n;
    size_t max_chunk = 0;
    for (int k = 0; k < K; k++) max_chunk = std::max(max_chunk, off[k + 1] - off[k]);

    struct Cleanup {   // every exit path: nothing in flight, nothing leaked
        DeviceCtx &c;
        void *d_bases = nullptr, *d_scalars = nullptr, *d_out = nullptr;
        std::vector<cudaEvent_t> ev;
        ~Cleanup() {
            cudaStreamSynchronize(c.copy_st);
            cudaStreamSynchronize(c.st);
            for (void *p : {d_bases, d_scalars, d_out})
                if (p) cudaFreeAsync(p, c.st);
            for (auto e : ev) cudaEventDestroy(e);
            cudaStreamSynchronize(c.st);
        }
    } cl{c};
    std::unique_ptr<MsmSessionBase> s(msm_session_create(curve));   // destroyed BEFORE cl: its frees are enqueued on c.st, then cl syncs
    cudaEvent_t alloc_done;
    AB_CUDA(cudaEventCreateWithFlags(&alloc_done, cudaEventDisableTiming));
    cl.ev.push_back(alloc_done);
    if (!d_bases_resident) AB_CUDA(cudaMallocAsync(&cl.d_bases, n * pb, c.st));
    AB_CUDA(cudaMallocAsync(&cl.d_scalars, n * sb, c.st));
    AB_CUDA(cudaMallocAsync(&cl.d_out, (size_t)3 * L * 4, c.st));
    AB_CUDA(cudaEventRecord(alloc_done, c.st));
    AB_CUDA(cudaStreamWaitEvent(c.copy_st, alloc_done, 0));
    const char *db = d_bases_resident ? (const char *)d_bases_resident : (const char *)cl.d_bases;
    if (int rc = s->begin(n, max_chunk, kind, c.st)) return rc;
    for (int k = 0; k < K; k++) {
        const size_t lo = off[k], cnt = off[k + 1] - off[k];
        cudaEvent_t ready;
        AB_CUDA(cudaEventCreateWithFlags(&ready, cudaEventDisableTiming));
        cl.ev.push_back(ready);
        if (int rc = h2d(c, (char *)cl.d_scalars + lo * sb, (const char *)scalars + lo * sb, cnt * sb)) return rc;
        if (!d_bases_resident)
            if (int rc = h2d(c, (char *)cl.d_bases + lo * pb, (const char *)bases + lo * pb, cnt * pb)) return rc;
        AB_CUDA(cudaEventRecord(ready, c.copy_st));
        if (int rc = s->add_chunk(db + lo * pb, (const char *)cl.d_scalars + lo * sb, cnt, ready)) return rc;
    }
    if (int rc = s->finish(cl.d_out)) return rc;
    AB_CUDA(cudaMemcpyAsync(out_xyz, cl.d_out, (size_t)3 * L * 4, cudaMemcpyDeviceToHost, c.st));
    AB_CUDA(cudaStreamSynchronize(c.st));
    return s->collect_timings();
}

static int check_msm_args(int curve, int kind, const void *bases, const void *scalars, size_t n, const void *out) {
    if (kind < B200_SCALARS_FR_MONT || kind > B200_SCALARS_U64) { set_last_error("unknown scalar kind"); return B200_EINVAL; }
    if (!msm_coord_words(curve)) { set_last_error("unknown curve id"); return B200_EINVAL; }
    if (!out || (n && (!bases || !scalars))) { set_last_error("null pointer"); return B200_EINVAL; }
    if (n >= ((size_t)1 << 31)) { set_last_error("n must be < 2^31 per device"); return B200_ETOOLARGE; }
    return 0;
}

// n pairs split into `parts` contiguous shards; shard d = [lo, hi)
static void shard(size_t n, int parts, int d, size_t *lo, size_t *hi) {
    const size_t base = n / parts, extra = n % parts;
    *lo = d * base + std::min<size_t>(d, extra);
    *hi = *lo + base + ((size_t)d < extra ? 1 : 0);
}

// run fn(d) on device d in its own host thread for d < ngpus; window / level settings of the calling thread are inherited
template <class Fn> static int per_device(int ngpus, Fn fn) {
    const int win = msm_get_window(), lev = msm_get_affine_levels();
    std::vector<int> rc((size_t)ngpus, 0);
    std::vector<std::string> msg((size_t)ngpus);
    auto body = [&](int d) {
        cudaError_t e = cudaSetDevice(d);
        if (e != cudaSuccess) { rc[d] = cuda_fail(e, "cudaSetDevice", __FILE__, __LINE__); }
        else {
            msm_set_window(win);
            msm_set_affine_levels(lev);
            rc[d] = ensure_device_init();
            if (!rc[d]) rc[d] = fn(d);
        }
        if (rc[d]) msg[d] = b200_last_error();
    };
    int dev0 = 0;
    cudaGetDevice(&dev0);
    int slice = 0, slices = 1;   // input-chunk sharding computes whole MSMs: the caller's bucket slice does not apply here
    msm_get_bucket_slice(&slice, &slices);
    msm_set_bucket_slice(0, 1);
    std::vector<std::thread> th;
    for (int d = 1; d < ngpus; d++) th.emplace_back(body, d);
    body(0);
    for (auto &t : th) t.join();
    msm_set_bucket_slice(slice, slices);
    cudaSetDevice(dev0);
    for (int d = 0; d < ngpus; d++)
        if (rc[d]) { set_last_error("device " + std::to_string(d) + ": " + msg[d]); return rc[d]; }
    return 0;
}
}  // namespace ab200
using namespace ab200;

struct b200_bases {
    int curve = 0, ngpus = 0;
    size_t n = 0;
    std::vector<void *> d_ptr;        // per device
    std::vector<size_t> lo, hi;       // shard of each device
};
struct b200_msm_stream {
    int curve = 0, kind = 0, dev = 0, pushes = 0;
    size_t max_chunk = 0;
    CtxLease lease;
    std::unique_ptr<MsmSessionBase> session;
    void *d_bases[2] = {nullptr, nullptr}, *d_scalars[2] = {nullptr, nullptr};
    cudaEvent_t consumed[2] = {nullptr, nullptr};   // recorded on the compute stream after the chunk in staging buffer i was accumulated
};

extern "C" {

int b200_msm_sw_g1_scalars_dev(int curve, int scalar_kind, const void *d_bases, const void *d_scalars, size_t n, uint64_t *out_xyz, void *stream) {
    { int irc = ensure_device_init(); if (irc) return irc; }
    return msm_dispatch(curve, scalar_kind, d_bases, d_scalars, n, out_xyz, (cudaStream_t)stream, 1, nullptr, nullptr);
}
int b200_msm_sw_g1_dev(int curve, const void *d_bases, const void *d_scalars, size_t n, uint64_t *out_xyz, void *stream) {
    return b200_msm_sw_g1_scalars_dev(curve, B200_SCALARS_FR_MONT, d_bases, d_scalars, n, out_xyz, stream);
}
int b200_msm_sw_g1(int curve, const uint64_t *bases, const uint64_t *scalars, size_t n, uint64_t *out_xyz) {
    return b200_msm_sw_g1_scalars(curve, B200_SCALARS_FR_MONT, bases, scalars, n, out_xyz);
}
int b200_msm_sw_g1_scalars(int curve, int scalar_kind, const uint64_t *bases, const void *scalars, size_t n, uint64_t *out_xyz) {
    { int irc = ensure_device_init(); if (irc) return irc; }
    if (int rc = check_msm_args(curve, scalar_kind, bases, scalars, n, out_xyz)) return rc;
    return host_msm(curve, scalar_kind, bases, nullptr, scalars, n, out_xyz);
}
int b200_msm_sw_g2(const uint64_t *bases, const uint64_t *scalars, size_t n, uint64_t *out_xyz) {
    return b200_msm_sw_g1_scalars(B200_CURVE_BLS12_381_G2, B200_SCALARS_FR_MONT, bases, scalars, n, out_xyz);
}
int b200_msm_sw_g2_dev(const void *d_bases, const void *d_scalars, size_t n, uint64_t *out_xyz, void *stream) {
    return b200_msm_sw_g1_scalars_dev(B200_CURVE_BLS12_381_G2, B200_SCALARS_FR_MONT, d_bases, d_scalars, n, out_xyz, stream);
}

int b200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

int b200_msm_sw_g1_multi(int curve, int ngpus, const uint64_t *bases, const uint64_t *scalars, size_t n, uint64_t *out_xyz) {
    if (int rc = check_msm_args(curve, B200_SCALARS_FR_MONT, bases, scalars, n / std::max(ngpus, 1), out_xyz)) return rc;
    if (ngpus < 1 || ngpus > b200_device_count()) { set_last_error("ngpus must be in [1, b200_device_count()]"); return B200_EINVAL; }
    const int L = msm_coord_words(curve);
    if (n == 0) { msm_write_zero(curve, out_xyz); return 0; }
    std::vector<uint64_t> partial((size_t)ngpus * 3 * L / 2);
    int rc = per_device(ngpus, [&](int d) {
        size_t lo, hi;
        shard(n, ngpus, d, &lo, &hi);
        return host_msm(curve, B200_SCALARS_FR_MONT, (const char *)bases + lo * (size_t)(2 * L * 4), nullptr, (const char *)scalars + lo * 32, hi - lo,
                        partial.data() + (size_t)d * 3 * L / 2);
    });
    if (rc) return rc;
    if (ngpus == 1) { memcpy(out_xyz, partial.data(), (size_t)3 * L * 4); return 0; }
    return g1_sum_dispatch(curve, partial.data(), (size_t)ngpus, out_xyz, false);
}

int b200_bases_upload(int curve, int ngpus, const uint64_t *bases, size_t n, b200_bases_t **handle) {
    const int L = msm_coord_words(curve);
    if (!L) { set_last_error("unknown curve id"); return B200_EINVAL; }
    if (!handle || (n && !bases)) { set_last_error("null pointer"); return B200_EINVAL; }
    if (ngpus < 1 || ngpus > b200_device_count()) { set_last_error("ngpus must be in [1, b200_device_count()]"); return B200_EINVAL; }
    std::unique_ptr<b200_bases> h(new b200_bases());
    h->curve = curve; h->ngpus = ngpus; h->n = n;
    h->d_ptr.assign((size_t)ngpus, nullptr); h->lo.resize((size_t)ngpus); h->hi.resize((size_t)ngpus);
    const size_t pb = (size_t)2 * L * 4;
    int rc = per_device(ngpus, [&](int d) {
        shard(n, ngpus, d, &h->lo[d], &h->hi[d]);
        const size_t cnt = h->hi[d] - h->lo[d];
        if (!cnt) return 0;
        CtxLease lease;
        if (int r = lease.acquire(d)) return r;
        AB_CUDA(cudaMalloc(&h->d_ptr[d], cnt * pb));
        int r = h2d(*lease.c, h->d_ptr[d], (const char *)bases + h->lo[d] * pb, cnt * pb);
        cudaError_t e = cudaStreamSynchronize(lease.c->copy_st);
        if (!r && e != cudaSuccess) r = cuda_fail(e, "cudaStreamSynchronize", __FILE__, __LINE__);
        return r;
    });
    if (rc) { b200_bases_free(h.release()); return rc; }
    *handle = h.release();
    return 0;
}
int b200_bases_free(b200_bases_t *h) {
    if (!h) return 0;
    int dev0 = 0;
    cudaGetDevice(&dev0);
    for (int d = 0; d < h->ngpus; d++)
        if (h->d_ptr[d]) { cudaSetDevice(d); cudaFree(h->d_ptr[d]); }
    cudaSetDevice(dev0);
    delete h;
    return 0;
}
int b200_msm_bases(const b200_bases_t *h, int scalar_kind, const void *scalars, size_t n, uint64_t *out_xyz) {
    if (!h) { set_last_error("null handle"); return B200_EINVAL; }
    if (n > h->n) { set_last_error("more scalars than uploaded bases"); return B200_EINVAL; }
    if (int rc = check_msm_args(h->curve, scalar_kind, scalars, scalars, n / (size_t)h->ngpus, out_xyz)) return rc;
    const int L = msm_coord_words(h->curve);
    if (n == 0) { msm_write_zero(h->curve, out_xyz); return 0; }
    const size_t sb = scalar_kind_bytes(scalar_kind);
    std::vector<uint64_t> partial((size_t)h->ngpus * 3 * L / 2);
    int rc = per_device(h->ngpus, [&](int d) {
        const size_t lo = std::min(n, h->lo[d]), hi = std::min(n, h->hi[d]);   // the first n bases
        return host_msm(h->curve, scalar_kind, nullptr, h->d_ptr[d], (const char *)scalars + lo * sb, hi - lo, partial.data() + (size_t)d * 3 * L / 2);
    });
    if (rc) return rc;
    if (h->ngpus == 1) { memcpy(out_xyz, partial.data(), (size_t)3 * L * 4); return 0; }
    return g1_sum_dispatch(h->curve, partial.data(), (size_t)h->ngpus, out_xyz, false);
}

int b200_msm_stream_begin(int curve, int scalar_kind, size_t n_total_hint, size_t max_chunk, b200_msm_stream_t **stream) {
    { int irc = ensure_device_init(); if (irc) return irc; }
    if (!stream || !max_chunk) { set_last_error("null handle pointer or max_chunk == 0"); return B200_EINVAL; }
    if (scalar_kind < B200_SCALARS_FR_MONT || scalar_kind > B200_SCALARS_U64) { set_last_error("unknown scalar kind"); return B200_EINVAL; }
    const int L = msm_coord_words(curve);
    if (!L) { set_last_error("unknown curve id"); return B200_EINVAL; }
    std::unique_ptr<b200_msm_stream> s(new b200_msm_stream());
    s->curve = curve; s->kind = scalar_kind; s->max_chunk = max_chunk;
    AB_CUDA(cudaGetDevice(&s->dev));
    if (int rc = s->lease.acquire(s->dev)) return rc;
    s->session.reset(msm_session_create(curve));
    DeviceCtx &c = *s->lease.c;
    int rc = s->session->begin(std::max(n_total_hint, max_chunk), max_chunk, scalar_kind, c.st);
    for (int i = 0; i < 2 && !rc; i++) {
        cudaError_t e = cudaMalloc(&s->d_bases[i], max_chunk * (size_t)(2 * L * 4));
        if (e == cudaSuccess) e = cudaMalloc(&s->d_scalars[i], max_chunk * scalar_kind_bytes(scalar_kind));
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&s->consumed[i], cudaEventDisableTiming);
        if (e != cudaSuccess) rc = cuda_fail(e, "stream staging allocation", __FILE__, __LINE__);
    }
    if (rc) { b200_msm_stream_abort(s.release()); return rc; }
    *stream = s.release();
    return 0;
}
int b200_msm_stream_push(b200_msm_stream_t *s, const uint64_t *bases, const void *scalars, size_t n) {
    if (!s) { set_last_error("null handle"); return B200_EINVAL; }
    if (n > s->max_chunk) { set_last_error("chunk larger than max_chunk"); return B200_EINVAL; }
    if (n == 0) return 0;
    if (!bases || !scalars) { set_last_error("null pointer"); return B200_EINVAL; }
    int dev = 0;
    AB_CUDA(cudaGetDevice(&dev));
    if (dev != s->dev) AB_CUDA(cudaSetDevice(s->dev));
    DeviceCtx &c = *s->lease.c;
    const int L = msm_coord_words(s->curve), b = s->pushes & 1;
    int rc = 0;
    cudaEvent_t ready = nullptr;
    cudaError_t e = cudaStreamWaitEvent(c.copy_st, s->consumed[b], 0);   // staging buffer b was last read by push k-2
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ready, cudaEventDisableTiming);
    if (e != cudaSuccess) rc = cuda_fail(e, "stream push", __FILE__, __LINE__);
    if (!rc) rc = h2d(c, s->d_scalars[b], scalars, n * scalar_kind_bytes(s->kind));
    if (!rc) rc = h2d(c, s->d_bases[b], bases, n * (size_t)(2 * L * 4));
    if (!rc) { e = cudaEventRecord(ready, c.copy_st); if (e != cudaSuccess) rc = cuda_fail(e, "cudaEventRecord", __FILE__, __LINE__); }
    if (!rc) rc = s->session->add_chunk(s->d_bases[b], s->d_scalars[b], n, ready);
    if (!rc) { e = cudaEventRecord(s->consumed[b], c.st); if (e != cudaSuccess) rc = cuda_fail(e, "cudaEventRecord", __FILE__, __LINE__); }
    // the caller may reuse its buffers as soon as push returns: wait for the copies (the arithmetic keeps running)
    e = cudaStreamSynchronize(c.copy_st);
    if (!rc && e != cudaSuccess) rc = cuda_fail(e, "cudaStreamSynchronize", __FILE__, __LINE__);
    if (ready) cudaEventDestroy(ready);
    s->pushes++;
    if (dev != s->dev) cudaSetDevice(dev);
    return rc;
}
int b200_msm_stream_abort(b200_msm_stream_t *s) {
    if (!s) return 0;
    int dev = 0;
    cudaGetDevice(&dev);
    cudaSetDevice(s->dev);
    if (s->lease.c) { cudaStreamSynchronize(s->lease.c->copy_st); cudaStreamSynchronize(s->lease.c->st); }
    s->session.reset();
    if (s->lease.c) cudaStreamSynchronize(s->lease.c->st);
    for (int i = 0; i < 2; i++) {
        if (s->d_bases[i]) cudaFree(s->d_bases[i]);
        if (s->d_scalars[i]) cudaFree(s->d_scalars[i]);
        if (s->consumed[i]) cudaEventDestroy(s->consumed[i]);
    }
    cudaSetDevice(dev);
    delete s;
    return 0;
}
int b200_msm_stream_finish(b200_msm_stream_t *s, uint64_t *out_xyz) {
    if (!s || !out_xyz) { set_last_error("null pointer"); if (s) b200_msm_stream_abort(s); return B200_EINVAL; }
    int dev = 0;
    cudaGetDevice(&dev);
    cudaSetDevice(s->dev);
    DeviceCtx &c = *s->lease.c;
    const int L = msm_coord_words(s->curve);
    void *d_out = nullptr;
    int rc = 0;
    cudaError_t e = cudaMallocAsync(&d_out, (size_t)3 * L * 4, c.st);
    if (e != cudaSuccess) rc = cuda_fail(e, "cudaMallocAsync", __FILE__, __LINE__);
    if (!rc) rc = s->session->finish(d_out);
    if (!rc) { e = cudaMemcpyAsync(out_xyz, d_out, (size_t)3 * L * 4, cudaMemcpyDeviceToHost, c.st); if (e != cudaSuccess) rc = cuda_fail(e, "cudaMemcpyAsync D2H", __FILE__, __LINE__); }
    if (d_out) cudaFreeAsync(d_out, c.st);
    e = cudaStreamSynchronize(c.st);
    if (!rc && e != cudaSuccess) rc = cuda_fail(e, "cudaStreamSynchronize", __FILE__, __LINE__);
    if (!rc) rc = s->session->collect_timings();
    cudaSetDevice(dev);
    b200_msm_stream_abort(s);
    return rc;
}

int b200_set_msm_window(int c) { return msm_set_window(c); }
int b200_set_msm_affine_levels(int levels) { return msm_set_affine_levels(levels); }
int b200_set_msm_bucket_slice(int slice, int slices) { return msm_set_bucket_slice(slice, slices); }
int b200_msm_window_for(int curve, size_t n) {
    if (!msm_coord_words(curve)) return B200_EINVAL;
    return msm_auto_window(n, curve == B200_CURVE_BN254 ? 254 : 255);
}
int b200_g1_sum(int curve, const uint64_t *points_xyz, size_t k, uint64_t *out_xyz) { if (int irc = ensure_device_init()) return irc; return g1_sum_dispatch(curve, points_xyz, k, out_xyz, false); }
int b200_g1_into_affine(int curve, const uint64_t *xyz, uint64_t *out_xy) { if (int irc = ensure_device_init()) return irc; return g1_sum_dispatch(curve, xyz, 1, out_xy, true); }

int b200_ntt_fr_dev(int field, void *d_data, uint32_t log_n, int inverse, const uint64_t *coset_offset, void *stream) {
    { int irc = ensure_device_init(); if (irc) return irc; }
    int rc = ntt_dispatch(field, d_data, log_n, inverse, coset_offset, (cudaStream_t)stream);
    if (rc) return rc;
    AB_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    return 0;
}

// host-buffer transform: H2D of the `len_in` given elements only (the zero padding of `fft_in_place`'s resize is produced on the
// device), transform, D2H of all 2^log_n results
int b200_ntt_fr_padded(int field, const uint64_t *in, size_t len_in, uint64_t *out, uint32_t log_n, int inverse, const uint64_t *coset_offset) {
    { int irc = ensure_device_init(); if (irc) return irc; }
    if (!out || (len_in && !in)) { set_last_error("null data pointer"); return B200_EINVAL; }
    if (field != B200_FIELD_BLS12_381_FR && field != B200_FIELD_BN254_FR) { set_last_error("unknown scalar field id"); return B200_EINVAL; }
    if (log_n > (uint32_t)(field == B200_FIELD_BLS12_381_FR ? 32 : 28)) {
        set_last_error("log_n exceeds TWO_ADICITY (Radix2EvaluationDomain::new would return None)");
        return B200_ETOOLARGE;
    }
    const size_t n = (size_t)1 << log_n, bytes = n * 32;
    if (len_in > n) len_in = n;   // coeffs.resize(self.size(), ..) truncates (radix2/mod.rs:144)
    int dev = 0;
    AB_CUDA(cudaGetDevice(&dev));
    CtxLease lease;
    if (int rc = lease.acquire(dev)) return rc;
    DeviceCtx &c = *lease.c;
    void *d = nullptr;
    AB_CUDA(cudaMallocAsync(&d, bytes, c.st));
    int rc = 0;
    cudaEvent_t ev = nullptr;
    cudaError_t e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventRecord(ev, c.st);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(c.copy_st, ev, 0);
    if (e != cudaSuccess) rc = cuda_fail(e, "event setup", __FILE__, __LINE__);
    if (!rc) rc = h2d(c, d, in, len_in * 32);                       // pinned: async; pageable: staged through the pinned ring
    if (!rc) { e = cudaEventRecord(ev, c.copy_st); if (e == cudaSuccess) e = cudaStreamWaitEvent(c.st, ev, 0); if (e != cudaSuccess) rc = cuda_fail(e, "event", __FILE__, __LINE__); }
    if (!rc && len_in < n) { e = cudaMemsetAsync((char *)d + len_in * 32, 0, (n - len_in) * 32, c.st); if (e != cudaSuccess) rc = cuda_fail(e, "cudaMemsetAsync", __FILE__, __LINE__); }
    if (!rc) rc = ntt_dispatch(field, d, log_n, inverse, coset_offset, c.st);
    if (!rc) { e = cudaMemcpyAsync(out, d, bytes, cudaMemcpyDeviceToHost, c.st); if (e != cudaSuccess) rc = cuda_fail(e, "cudaMemcpyAsync D2H", __FILE__, __LINE__); }
    cudaStreamSynchronize(c.copy_st);
    cudaFreeAsync(d, c.st);
    e = cudaStreamSynchronize(c.st);
    if (!rc && e != cudaSuccess) rc = cuda_fail(e, "cudaStreamSynchronize", __FILE__, __LINE__);
    if (ev) cudaEventDestroy(ev);
    return rc;
}
int b200_ntt_fr(int field, uint64_t *data, uint32_t log_n, int inverse, const uint64_t *coset_offset) {
    return b200_ntt_fr_padded(field, data, log_n <= 40 ? (size_t)1 << log_n : 0, data, log_n, inverse, coset_offset);
}
int b200_ntt_g1_dev(int curve, void *d_points, uint32_t log_n, int inverse, const uint64_t *coset_offset, void *stream) {
    { int irc = ensure_device_init(); if (irc) return irc; }
    int rc = point_ntt_dispatch(curve, d_points, log_n, inverse, coset_offset, (cudaStream_t)stream);
    if (rc) return rc;
    AB_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    return 0;
}
// host-buffer point transform: staged H2D (pinned or pageable), transform in place on the device, D2H
int b200_ntt_g1(int curve, uint64_t *points, uint32_t log_n, int inverse, const uint64_t *coset_offset) {
    { int irc = ensure_device_init(); if (irc) return irc; }
    if (int rc = point_ntt_check(curve, points, log_n)) return rc;
    const size_t bytes = ((size_t)1 << log_n) * 3 * (size_t)point_ntt_coord_words(curve) * 4;
    int dev = 0;
    AB_CUDA(cudaGetDevice(&dev));
    CtxLease lease;
    if (int rc = lease.acquire(dev)) return rc;
    DeviceCtx &c = *lease.c;
    void *d = nullptr;
    AB_CUDA(cudaMallocAsync(&d, bytes, c.st));
    int rc = 0;
    cudaEvent_t ev = nullptr;
    cudaError_t e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventRecord(ev, c.st);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(c.copy_st, ev, 0);
    if (e != cudaSuccess) rc = cuda_fail(e, "event setup", __FILE__, __LINE__);
    if (!rc) rc = h2d(c, d, points, bytes);
    if (!rc) { e = cudaEventRecord(ev, c.copy_st); if (e == cudaSuccess) e = cudaStreamWaitEvent(c.st, ev, 0); if (e != cudaSuccess) rc = cuda_fail(e, "event", __FILE__, __LINE__); }
    if (!rc) rc = point_ntt_dispatch(curve, d, log_n, inverse, coset_offset, c.st);
    if (!rc) { e = cudaMemcpyAsync(points, d, bytes, cudaMemcpyDeviceToHost, c.st); if (e != cudaSuccess) rc = cuda_fail(e, "cudaMemcpyAsync D2H", __FILE__, __LINE__); }
    cudaStreamSynchronize(c.copy_st);
    cudaFreeAsync(d, c.st);
    e = cudaStreamSynchronize(c.st);
    if (!rc && e != cudaSuccess) rc = cuda_fail(e, "cudaStreamSynchronize", __FILE__, __LINE__);
    if (ev) cudaEventDestroy(ev);
    return rc;
}
int b200_clear_cache(void) {
    int rc = ntt_clear_cache();
    // also hand the stream-ordered scratch retained by the default memory pool back to the driver (a 2^26 MSM keeps tens
    // of GB of level buffers cached for the next call otherwise)
    int dev = 0;
    cudaMemPool_t pool;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
        cudaDeviceSynchronize();
        cudaMemPoolTrimTo(pool, 0);
    }
    return rc;
}

size_t b200_poly_mul_size(int field, size_t la, size_t lb) {
    if ((field != B200_FIELD_BLS12_381_FR && field != B200_FIELD_BN254_FR) || la == 0 || lb == 0) return 0;
    const size_t need = la + lb - 1;
    size_t n = 1;
    uint32_t lg = 0;
    while (n < need) { n <<= 1; lg++; }
    return lg > (uint32_t)(field == B200_FIELD_BLS12_381_FR ? 32 : 28) ? 0 : n;
}

static int poly_mul_on_device(int field, const void *d_a, size_t la, const void *d_b, size_t lb, void *d_out, cudaStream_t st) {
    const size_t n = b200_poly_mul_size(field, la, lb);
    if (!n) { set_last_error("empty operand or product degree past TWO_ADICITY"); return la && lb ? B200_ETOOLARGE : B200_EINVAL; }
    uint32_t lg = 0;
    while (((size_t)1 << lg) < n) lg++;
    void *tmp = nullptr;
    AB_CUDA(cudaMallocAsync(&tmp, n * 32, st));
    // evaluate_over_domain: zero-pad to n, forward transform
    AB_CUDA(cudaMemsetAsync(d_out, 0, n * 32, st));
    AB_CUDA(cudaMemsetAsync(tmp, 0, n * 32, st));
    AB_CUDA(cudaMemcpyAsync(d_out, d_a, la * 32, cudaMemcpyDeviceToDevice, st));
    AB_CUDA(cudaMemcpyAsync(tmp, d_b, lb * 32, cudaMemcpyDeviceToDevice, st));
    int rc = ntt_dispatch(field, d_out, lg, 0, nullptr, st);
    if (!rc) rc = ntt_dispatch(field, tmp, lg, 0, nullptr, st);
    // self_evals *= &other_evals ; interpolate
    if (!rc) rc = fp_op_dispatch(field == B200_FIELD_BLS12_381_FR ? 1 : 3, 0, d_out, tmp, d_out, n, 1, st);
    if (!rc) rc = ntt_dispatch(field, d_out, lg, 1, nullptr, st);
    cudaFreeAsync(tmp, st);
    return rc;
}

int b200_poly_mul_fr_dev(int field, const void *d_a, size_t la, const void *d_b, size_t lb, void *d_out, void *stream) {
    { int irc = ensure_device_init(); if (irc) return irc; }
    if (!d_a || !d_b || !d_out) { set_last_error("null pointer"); return B200_EINVAL; }
    int rc = poly_mul_on_device(field, d_a, la, d_b, lb, d_out, (cudaStream_t)stream);
    if (rc) return rc;
    AB_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    return 0;
}

int b200_poly_mul_fr(int field, const uint64_t *a, size_t la, const uint64_t *b, size_t lb, uint64_t *out) {
    { int irc = ensure_device_init(); if (irc) return irc; }
    if (!a || !b || !out) { set_last_error("null pointer"); return B200_EINVAL; }
    const size_t n = b200_poly_mul_size(field, la, lb);
    if (!n) { set_last_error("empty operand or product degree past TWO_ADICITY"); return la && lb ? B200_ETOOLARGE : B200_EINVAL; }
    cudaStream_t st = 0;
    void *d_a = nullptr, *d_b = nullptr, *d_o = nullptr;
    AB_CUDA(cudaMallocAsync(&d_a, la * 32, st));
    AB_CUDA(cudaMallocAsync(&d_b, lb * 32, st));
    AB_CUDA(cudaMallocAsync(&d_o, n * 32, st));
    AB_CUDA(cudaMemcpyAsync(d_a, a, la * 32, cudaMemcpyHostToDevice, st));
    AB_CUDA(cudaMemcpyAsync(d_b, b, lb * 32, cudaMemcpyHostToDevice, st));
    int rc = poly_mul_on_device(field, d_a, la, d_b, lb, d_o, st);
    if (!rc) {
        cudaError_t e = cudaMemcpyAsync(out, d_o, n * 32, cudaMemcpyDeviceToHost, st);
        if (e != cudaSuccess) rc = cuda_fail(e, "cudaMemcpyAsync D2H", __FILE__, __LINE__);
    }
    cudaFreeAsync(d_a, st); cudaFreeAsync(d_b, st); cudaFreeAsync(d_o, st);
    cudaError_t e = cudaStreamSynchronize(st);
    if (!rc && e != cudaSuccess) rc = cuda_fail(e, "cudaStreamSynchronize", __FILE__, __LINE__);
    return rc;
}

int b200_gen_bases_dev(int curve, uint64_t seed, size_t n, void *d_bases, void *d_b, void *stream) {
    { int irc = ensure_device_init(); if (irc) return irc; }
    int rc = gen_bases_dispatch(curve, seed, n, d_bases, d_b, (cudaStream_t)stream);
    if (rc) return rc;
    AB_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    return 0;
}
int b200_gen_scalars_dev(int field, uint64_t seed, size_t n, void *d_scalars, void *stream) {
    { int irc = ensure_device_init(); if (irc) return irc; }
    int rc = gen_scalars_dispatch(field, seed, n, d_scalars, (cudaStream_t)stream);
    if (rc) return rc;
    AB_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    return 0;
}
int b200_g1_batch_mul_dev(int curve, const uint64_t *base_xy, const void *d_scalars, size_t n, void *d_out_xy, void *stream) {
    { int irc = ensure_device_init(); if (irc) return irc; }
    int rc = batch_mul_dispatch(curve, base_xy, d_scalars, n, d_out_xy, (cudaStream_t)stream);
    if (rc) return rc;
    AB_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    return 0;
}
int b200_g1_normalize_batch_dev(int curve, const void *d_xyz, size_t n, void *d_out_xy, void *stream) {
    { int irc = ensure_device_init(); if (irc) return irc; }
    int rc = normalize_batch_dispatch(curve, d_xyz, n, d_out_xy, (cudaStream_t)stream);
    if (rc) return rc;
    AB_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    return 0;
}
int b200_fp_op_dev(int field, int op, const void *d_a, const void *d_b, void *d_out, size_t n, int reps, void *stream) {
    { int irc = ensure_device_init(); if (irc) return irc; }
    int rc = fp_op_dispatch(field, op, d_a, d_b, d_out, n, reps, (cudaStream_t)stream);
    if (rc) return rc;
    AB_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    return 0;
}
int b200_ec_op_dev(int curve, int op, const void *d_a, const void *d_b, void *d_out, size_t n, void *stream) {
    { int irc = ensure_device_init(); if (irc) return irc; }
    int rc = ec_op_dispatch(curve, op, d_a, d_b, d_out, n, (cudaStream_t)stream);
    if (rc) return rc;
    AB_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    return 0;
}
int b200_msm_last_timings(float *ms7, int *c, int *windows, unsigned long long *bucket_adds) { return msm_last_timings(ms7, c, windows, bucket_adds); }

}  // extern "C"
