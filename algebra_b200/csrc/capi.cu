// capi.cu — the extern "C" boundary declared in include/algebra_b200.h.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>
#include "common.cuh"
#include "host_api.h"

namespace ab200 {
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

// One call with host buffers on the CURRENT device: the leased context `c`, the call's stream-ordered scratch and its events.
// Uploads run on c->copy_st, the compute and the downloads on c->st.  On every exit path the destructor synchronises both
// streams before it frees anything: nothing of the call is in flight when it returns, and the caller may reuse its buffers.
struct HostCall {
    CtxLease lease;
    DeviceCtx *c = nullptr;
    std::vector<void *> mem;
    std::vector<cudaEvent_t> ev;
    bool alloc_pending = false;   // scratch allocated on c->st that c->copy_st is not yet ordered after

    int begin() {
        int dev = 0;
        AB_CUDA(cudaGetDevice(&dev));
        if (int rc = lease.acquire(dev)) return rc;
        c = lease.c;
        return 0;
    }
    template <class T> int alloc(T **p, size_t bytes) {
        void *q = nullptr;
        AB_CUDA(cudaMallocAsync(&q, bytes ? bytes : 16, c->st));
        mem.push_back(q);
        *p = (T *)q;
        alloc_pending = true;
        return 0;
    }
    // device dst <- host src through h2d, after the scratch allocated so far
    int upload(void *dst, const void *src, size_t bytes) {
        if (alloc_pending) {
            cudaEvent_t e;
            if (int rc = event(&e)) return rc;
            AB_CUDA(cudaEventRecord(e, c->st));
            AB_CUDA(cudaStreamWaitEvent(c->copy_st, e, 0));
            alloc_pending = false;
        }
        return h2d(*c, dst, src, bytes);
    }
    // *done fires when every upload so far has landed
    int uploaded(cudaEvent_t *done) {
        if (int rc = event(done)) return rc;
        AB_CUDA(cudaEventRecord(*done, c->copy_st));
        return 0;
    }
    int wait_uploads() {   // c->st waits for every upload so far
        cudaEvent_t done;
        if (int rc = uploaded(&done)) return rc;
        AB_CUDA(cudaStreamWaitEvent(c->st, done, 0));
        return 0;
    }
    int download(void *dst, const void *src, size_t bytes) {
        cudaError_t e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c->st);
        return e == cudaSuccess ? 0 : cuda_fail(e, "cudaMemcpyAsync D2H", __FILE__, __LINE__);
    }
    int sync() {   // the result of a successful call is on the host
        cudaError_t e = cudaStreamSynchronize(c->st);
        return e == cudaSuccess ? 0 : cuda_fail(e, "cudaStreamSynchronize", __FILE__, __LINE__);
    }
    ~HostCall() {
        if (!c) return;
        cudaStreamSynchronize(c->copy_st);
        cudaStreamSynchronize(c->st);
        for (void *p : mem) cudaFreeAsync(p, c->st);
        for (cudaEvent_t e : ev) cudaEventDestroy(e);
        cudaStreamSynchronize(c->st);
    }

private:
    int event(cudaEvent_t *e) {
        AB_CUDA(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
        ev.push_back(*e);
        return 0;
    }
};

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
    if (n == 0) { msm_write_zero(curve, out_xyz); return 0; }
    HostCall h;
    if (int rc = h.begin()) return rc;
    const size_t sb = scalar_kind_bytes(kind), pb = (size_t)2 * curve_info(curve)->coord_words * 4;
    const ChunkPlan &plan = chunk_plan();
    const int K = n >= ((size_t)1 << 22) ? plan.K : 1;
    size_t off[9];
    for (int k = 0; k <= K; k++) off[k] = K == 1 ? (size_t)k * n : n / 16 * (size_t)plan.bounds[k];
    off[K] = n;
    size_t max_chunk = 0;
    for (int k = 0; k < K; k++) max_chunk = std::max(max_chunk, off[k + 1] - off[k]);

    std::unique_ptr<MsmSessionBase> s(msm_session_create(curve));   // destroyed BEFORE h: its frees are enqueued on c->st, then h syncs
    char *d_bases = nullptr, *d_scalars = nullptr;
    if (!d_bases_resident)
        if (int rc = h.alloc(&d_bases, n * pb)) return rc;
    if (int rc = h.alloc(&d_scalars, n * sb)) return rc;
    const char *db = d_bases_resident ? (const char *)d_bases_resident : d_bases;
    if (int rc = s->begin(n, max_chunk, kind, h.c->st)) return rc;
    for (int k = 0; k < K; k++) {
        const size_t lo = off[k], cnt = off[k + 1] - off[k];
        if (int rc = h.upload(d_scalars + lo * sb, (const char *)scalars + lo * sb, cnt * sb)) return rc;
        if (!d_bases_resident)
            if (int rc = h.upload(d_bases + lo * pb, (const char *)bases + lo * pb, cnt * pb)) return rc;
        cudaEvent_t ready;
        if (int rc = h.uploaded(&ready)) return rc;
        if (int rc = s->add_chunk(db + lo * pb, d_scalars + lo * sb, cnt, ready)) return rc;
    }
    return msm_session_result(*s, out_xyz, h.c->st);
}

static int check_msm_args(int curve, int kind, const void *bases, const void *scalars, size_t n, const void *out) {
    if (int rc = check_scalar_kind(kind)) return rc;
    if (!curve_info(curve)) { set_last_error("unknown curve id"); return B200_EINVAL; }
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

// host points in, host result out: the sum of k Jacobian points, or (to_affine) the affine form of each of the k points
static int host_g1_sum(int curve, const uint64_t *pts, size_t k, uint64_t *out, bool to_affine) {
    const CurveInfo *ci = curve_info(curve);
    if (!ci) { set_last_error("unknown curve id"); return B200_EINVAL; }
    if (!pts || !out) { set_last_error("null pointer"); return B200_EINVAL; }
    const size_t L = (size_t)ci->coord_words, in_bytes = k * 3 * L * 4, out_bytes = (to_affine ? k * 2 * L : 3 * L) * 4;
    HostCall h;
    void *d_in = nullptr, *d_out = nullptr;
    if (int rc = h.begin()) return rc;
    if (int rc = h.alloc(&d_in, in_bytes)) return rc;
    if (int rc = h.alloc(&d_out, out_bytes)) return rc;
    if (int rc = h.upload(d_in, pts, in_bytes)) return rc;
    if (int rc = h.wait_uploads()) return rc;
    if (int rc = g1_sum(curve, d_in, k, d_out, to_affine, h.c->st)) return rc;
    if (int rc = h.download(out, d_out, out_bytes)) return rc;
    return h.sync();
}

// one MSM split over ngpus devices: part(d, partial) computes device d's Jacobian result into `partial`; the partial results
// are then added on the current device
template <class Fn> static int msm_over_devices(int curve, int ngpus, uint64_t *out_xyz, Fn part) {
    const size_t words = (size_t)3 * curve_info(curve)->coord_words / 2;   // u64 per Jacobian point
    std::vector<uint64_t> partial((size_t)ngpus * words);
    if (int rc = per_device(ngpus, [&](int d) { return part(d, partial.data() + (size_t)d * words); })) return rc;
    if (ngpus == 1) { memcpy(out_xyz, partial.data(), words * 8); return 0; }
    return host_g1_sum(curve, partial.data(), (size_t)ngpus, out_xyz, false);
}

// the device-buffer entry points: dispatch(st) on the caller's stream, then wait for it
template <class Fn> static int on_stream(void *stream, Fn dispatch) {
    if (int rc = ensure_device_init()) return rc;
    if (int rc = dispatch((cudaStream_t)stream)) return rc;
    AB_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
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
    if (n == 0) { msm_write_zero(curve, out_xyz); return 0; }
    const size_t pb = (size_t)2 * curve_info(curve)->coord_words * 4;
    return msm_over_devices(curve, ngpus, out_xyz, [&](int d, uint64_t *partial) {
        size_t lo, hi;
        shard(n, ngpus, d, &lo, &hi);
        return host_msm(curve, B200_SCALARS_FR_MONT, (const char *)bases + lo * pb, nullptr, (const char *)scalars + lo * 32, hi - lo, partial);
    });
}

int b200_bases_upload(int curve, int ngpus, const uint64_t *bases, size_t n, b200_bases_t **handle) {
    const CurveInfo *ci = curve_info(curve);
    if (!ci) { set_last_error("unknown curve id"); return B200_EINVAL; }
    if (!handle || (n && !bases)) { set_last_error("null pointer"); return B200_EINVAL; }
    if (ngpus < 1 || ngpus > b200_device_count()) { set_last_error("ngpus must be in [1, b200_device_count()]"); return B200_EINVAL; }
    std::unique_ptr<b200_bases> h(new b200_bases());
    h->curve = curve; h->ngpus = ngpus; h->n = n;
    h->d_ptr.assign((size_t)ngpus, nullptr); h->lo.resize((size_t)ngpus); h->hi.resize((size_t)ngpus);
    const size_t pb = (size_t)2 * ci->coord_words * 4;
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
    if (n == 0) { msm_write_zero(h->curve, out_xyz); return 0; }
    const size_t sb = scalar_kind_bytes(scalar_kind);
    return msm_over_devices(h->curve, h->ngpus, out_xyz, [&](int d, uint64_t *partial) {
        const size_t lo = std::min(n, h->lo[d]), hi = std::min(n, h->hi[d]);   // the first n bases
        return host_msm(h->curve, scalar_kind, nullptr, h->d_ptr[d], (const char *)scalars + lo * sb, hi - lo, partial);
    });
}

int b200_msm_stream_begin(int curve, int scalar_kind, size_t n_total_hint, size_t max_chunk, b200_msm_stream_t **stream) {
    { int irc = ensure_device_init(); if (irc) return irc; }
    if (!stream || !max_chunk) { set_last_error("null handle pointer or max_chunk == 0"); return B200_EINVAL; }
    if (int rc = check_scalar_kind(scalar_kind)) return rc;
    const CurveInfo *ci = curve_info(curve);
    if (!ci) { set_last_error("unknown curve id"); return B200_EINVAL; }
    std::unique_ptr<b200_msm_stream> s(new b200_msm_stream());
    s->curve = curve; s->kind = scalar_kind; s->max_chunk = max_chunk;
    AB_CUDA(cudaGetDevice(&s->dev));
    if (int rc = s->lease.acquire(s->dev)) return rc;
    s->session.reset(msm_session_create(curve));
    DeviceCtx &c = *s->lease.c;
    int rc = s->session->begin(std::max(n_total_hint, max_chunk), max_chunk, scalar_kind, c.st);
    for (int i = 0; i < 2 && !rc; i++) {
        cudaError_t e = cudaMalloc(&s->d_bases[i], max_chunk * (size_t)(2 * ci->coord_words * 4));
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
    const int L = curve_info(s->curve)->coord_words, b = s->pushes & 1;
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
    const int rc = msm_session_result(*s->session, out_xyz, s->lease.c->st);
    cudaSetDevice(dev);
    b200_msm_stream_abort(s);
    return rc;
}

int b200_set_msm_window(int c) { return msm_set_window(c); }
int b200_set_msm_affine_levels(int levels) { return msm_set_affine_levels(levels); }
int b200_set_msm_bucket_slice(int slice, int slices) { return msm_set_bucket_slice(slice, slices); }
int b200_msm_window_for(int curve, size_t n) {
    const CurveInfo *ci = curve_info(curve);
    if (!ci) return B200_EINVAL;
    return msm_auto_window(n, ci->scalar_bits);
}
int b200_g1_sum(int curve, const uint64_t *points_xyz, size_t k, uint64_t *out_xyz) { if (int irc = ensure_device_init()) return irc; return host_g1_sum(curve, points_xyz, k, out_xyz, false); }
int b200_g1_into_affine(int curve, const uint64_t *xyz, uint64_t *out_xy) { if (int irc = ensure_device_init()) return irc; return host_g1_sum(curve, xyz, 1, out_xy, true); }

int b200_ntt_fr_dev(int field, void *d_data, uint32_t log_n, int inverse, const uint64_t *coset_offset, void *stream) {
    return on_stream(stream, [&](cudaStream_t st) { return ntt_dispatch(field, d_data, log_n, inverse, coset_offset, st); });
}

// host-buffer transform: H2D of the `len_in` given elements only (the zero padding of `fft_in_place`'s resize is produced on the
// device), transform, D2H of all 2^log_n results
int b200_ntt_fr_padded(int field, const uint64_t *in, size_t len_in, uint64_t *out, uint32_t log_n, int inverse, const uint64_t *coset_offset) {
    { int irc = ensure_device_init(); if (irc) return irc; }
    if (!out || (len_in && !in)) { set_last_error("null data pointer"); return B200_EINVAL; }
    const FieldInfo *fi = field_info(field);
    if (!fi) { set_last_error("unknown scalar field id"); return B200_EINVAL; }
    if (log_n > (uint32_t)fi->two_adicity) {
        set_last_error("log_n exceeds TWO_ADICITY (Radix2EvaluationDomain::new would return None)");
        return B200_ETOOLARGE;
    }
    const size_t n = (size_t)1 << log_n, bytes = n * 32;
    if (len_in > n) len_in = n;   // coeffs.resize(self.size(), ..) truncates (radix2/mod.rs:144)
    HostCall h;
    char *d = nullptr;
    if (int rc = h.begin()) return rc;
    if (int rc = h.alloc(&d, bytes)) return rc;
    if (int rc = h.upload(d, in, len_in * 32)) return rc;   // in == out (b200_ntt_fr): the D2H below is ordered after this upload
    if (int rc = h.wait_uploads()) return rc;
    if (len_in < n) AB_CUDA(cudaMemsetAsync(d + len_in * 32, 0, (n - len_in) * 32, h.c->st));
    if (int rc = ntt_dispatch(field, d, log_n, inverse, coset_offset, h.c->st)) return rc;
    if (int rc = h.download(out, d, bytes)) return rc;
    return h.sync();
}
int b200_ntt_fr(int field, uint64_t *data, uint32_t log_n, int inverse, const uint64_t *coset_offset) {
    return b200_ntt_fr_padded(field, data, log_n <= 40 ? (size_t)1 << log_n : 0, data, log_n, inverse, coset_offset);
}
int b200_ntt_g1_dev(int curve, void *d_points, uint32_t log_n, int inverse, const uint64_t *coset_offset, void *stream) {
    return on_stream(stream, [&](cudaStream_t st) { return point_ntt_dispatch(curve, d_points, log_n, inverse, coset_offset, st); });
}
// host-buffer point transform: staged H2D (pinned or pageable), transform in place on the device, D2H
int b200_ntt_g1(int curve, uint64_t *points, uint32_t log_n, int inverse, const uint64_t *coset_offset) {
    { int irc = ensure_device_init(); if (irc) return irc; }
    if (int rc = point_ntt_check(curve, points, log_n)) return rc;
    const size_t bytes = ((size_t)1 << log_n) * 3 * (size_t)curve_info(curve)->coord_words * 4;
    HostCall h;
    void *d = nullptr;
    if (int rc = h.begin()) return rc;
    if (int rc = h.alloc(&d, bytes)) return rc;
    if (int rc = h.upload(d, points, bytes)) return rc;
    if (int rc = h.wait_uploads()) return rc;
    if (int rc = point_ntt_dispatch(curve, d, log_n, inverse, coset_offset, h.c->st)) return rc;
    if (int rc = h.download(points, d, bytes)) return rc;
    return h.sync();
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
    const FieldInfo *fi = field_info(field);
    if (!fi || la == 0 || lb == 0) return 0;
    const size_t need = la + lb - 1;
    size_t n = 1;
    uint32_t lg = 0;
    while (n < need) { n <<= 1; lg++; }
    return lg > (uint32_t)fi->two_adicity ? 0 : n;
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
    if (!rc) rc = fp_op_dispatch(field_info(field)->fp_op_field, 0, d_out, tmp, d_out, n, 1, st);
    if (!rc) rc = ntt_dispatch(field, d_out, lg, 1, nullptr, st);
    cudaFreeAsync(tmp, st);
    return rc;
}

int b200_poly_mul_fr_dev(int field, const void *d_a, size_t la, const void *d_b, size_t lb, void *d_out, void *stream) {
    return on_stream(stream, [&](cudaStream_t st) {
        if (!d_a || !d_b || !d_out) { set_last_error("null pointer"); return B200_EINVAL; }
        return poly_mul_on_device(field, d_a, la, d_b, lb, d_out, st);
    });
}

int b200_poly_mul_fr(int field, const uint64_t *a, size_t la, const uint64_t *b, size_t lb, uint64_t *out) {
    { int irc = ensure_device_init(); if (irc) return irc; }
    if (!a || !b || !out) { set_last_error("null pointer"); return B200_EINVAL; }
    const size_t n = b200_poly_mul_size(field, la, lb);
    if (!n) { set_last_error("empty operand or product degree past TWO_ADICITY"); return la && lb ? B200_ETOOLARGE : B200_EINVAL; }
    HostCall h;
    void *d_a = nullptr, *d_b = nullptr, *d_o = nullptr;
    if (int rc = h.begin()) return rc;
    if (int rc = h.alloc(&d_a, la * 32)) return rc;
    if (int rc = h.alloc(&d_b, lb * 32)) return rc;
    if (int rc = h.alloc(&d_o, n * 32)) return rc;
    if (int rc = h.upload(d_a, a, la * 32)) return rc;
    if (int rc = h.upload(d_b, b, lb * 32)) return rc;
    if (int rc = h.wait_uploads()) return rc;
    if (int rc = poly_mul_on_device(field, d_a, la, d_b, lb, d_o, h.c->st)) return rc;
    if (int rc = h.download(out, d_o, n * 32)) return rc;
    return h.sync();
}

int b200_gen_bases_dev(int curve, uint64_t seed, size_t n, void *d_bases, void *d_b, void *stream) {
    return on_stream(stream, [&](cudaStream_t st) { return gen_bases_dispatch(curve, seed, n, d_bases, d_b, st); });
}
int b200_gen_scalars_dev(int field, uint64_t seed, size_t n, void *d_scalars, void *stream) {
    return on_stream(stream, [&](cudaStream_t st) { return gen_scalars_dispatch(field, seed, n, d_scalars, st); });
}
int b200_g1_batch_mul_dev(int curve, const uint64_t *base_xy, const void *d_scalars, size_t n, void *d_out_xy, void *stream) {
    return on_stream(stream, [&](cudaStream_t st) { return batch_mul_dispatch(curve, base_xy, d_scalars, n, d_out_xy, st); });
}
int b200_g1_normalize_batch_dev(int curve, const void *d_xyz, size_t n, void *d_out_xy, void *stream) {
    return on_stream(stream, [&](cudaStream_t st) { return normalize_batch_dispatch(curve, d_xyz, n, d_out_xy, st); });
}
int b200_fp_op_dev(int field, int op, const void *d_a, const void *d_b, void *d_out, size_t n, int reps, void *stream) {
    return on_stream(stream, [&](cudaStream_t st) { return fp_op_dispatch(field, op, d_a, d_b, d_out, n, reps, st); });
}
int b200_ec_op_dev(int curve, int op, const void *d_a, const void *d_b, void *d_out, size_t n, void *stream) {
    return on_stream(stream, [&](cudaStream_t st) { return ec_op_dispatch(curve, op, d_a, d_b, d_out, n, st); });
}
int b200_msm_last_timings(float *ms7, int *c, int *windows, unsigned long long *bucket_adds) { return msm_last_timings(ms7, c, windows, bucket_adds); }

}  // extern "C"
