// cfb_pool.cu -- asynchronous, in-order, multi-GPU frame pool (see include/cfhd_b200.h).
//
// GPU re-hosting of the reference's CEncoderPool / EncoderJobQueue (EncoderSDK/EncoderPool.cpp:239,
// EncoderQueue.h:311-352): same contract (bounded queue, round-robin assignment, strict in-order delivery,
// borrowed buffers), but a "worker" is a GPU, not a CPU thread running the SSE2 transform.  Frames are
// independent, so GPUs never exchange data (no NCCL, SURVEY 8e).
//
// Per GPU: ONE issuing thread and ONE completing thread drive
//     upload streams (H2D copy engine)  ->  one compute stream per slot (SMs)  ->  download streams (D2H copy engine)
// chained by events, over `slots` sets of device staging.  The issuer takes up to `batch` queued jobs of its GPU,
// enqueues their uploads, the kernels (gated by the upload event) and the downloads (gated by the kernel event)
// without ever waiting for the GPU, so uploads of job k+1, kernels of job k and downloads of job k-1 overlap and both
// PCIe directions stay busy; the completer sleeps on the download event of the oldest slot in flight (blocking-sync
// events: the GPU boxes run under a CPU quota, spinning threads would throttle the caller), fetches the tail of a
// sparse result whose value count exceeded the speculative copy, publishes the jobs and recycles the slot.
// (Round 1 used one blocking thread per slot -- 16 per GPU -- each doing upload, kernels, download synchronously on
// one stream; at 8 GPUs that was 128 threads fighting over 16-24 usable cores.)
#include <algorithm>
#include <condition_variable>
#include <deque>
#include <memory>
#include <mutex>
#include <new>
#include <thread>
#include <vector>

#include "cfb_host.h"

using namespace cfb;

namespace {

struct Job {
    uint32_t frame_number = 0;
    bool inverse = false;
    bool sparse = false;
    const void *src = nullptr;
    void *dst = nullptr;
    int pitch = 0;
    int out_format = 0;
    cfb_quant quant{};
    int device_index = 0;
    bool taken = false, done = false;
    int overtaken = 0;                      // younger jobs of the other direction issued before this one
    cfb_error error = CFB_OK;
};

constexpr int kMaxOvertake = 8;

constexpr int kCopyStreams = 2;

struct Slot {
    int lane = 0;                           // which of the device's copy-stream pairs this slot uses
    cfb_context *ctx = nullptr;             // own compute stream: the kernels of a job wait for THAT job's upload only
    cfb_codec *codec = nullptr;             // device staging for `batch` frames (frames, pyramids, sparse buffers)
    cudaEvent_t ev_up = nullptr, ev_k = nullptr, ev_down = nullptr;
    std::vector<std::shared_ptr<Job>> jobs;
    unsigned guess = 0;                     // bytes copied speculatively for the sparse results of this batch
    uint64_t up_bytes = 0, down_bytes = 0;  // PCIe bytes of this batch in either direction (estimates, for the issue balance)
    cfb_error issue_error = CFB_OK;
};

struct Device {
    int device = 0, index = 0;
    // kCopyStreams streams per direction, slots alternate between them: two copies of one direction in flight keep the
    // link busy across copy boundaries (tools/pcie_pattern.py measures the effect)
    cudaStream_t s_up[kCopyStreams] = {}, s_down[kCopyStreams] = {};
    std::vector<std::unique_ptr<Slot>> slots;
    std::deque<int> free_slots;             // guarded by cfb_pool::mu
    std::deque<int> in_flight;              // issue order, guarded by cfb_pool::mu
    std::condition_variable cv_flight;
    unsigned value_guess = 0;               // running estimate of a frame's sparse size in bytes (all slots of this GPU)
    uint64_t up_pending = 0, down_pending = 0;  // bytes issued and not yet delivered, per PCIe direction (guarded by mu)
    bool issuer_done = false;               // guarded by cfb_pool::mu: nothing more will enter in_flight
    std::thread issuer, completer;
};

}  // namespace

struct cfb_pool {
    cfb_frame_desc desc{};
    cfb_layout layout{};
    int batch = 1, queue_length = 1;
    std::vector<int> devices;
    std::vector<std::unique_ptr<Device>> devs;

    std::mutex mu;
    std::condition_variable cv_work, cv_done, cv_space;
    std::deque<std::shared_ptr<Job>> queue;         // submission order; front = oldest undelivered
    uint64_t submitted = 0;
    bool stopping = false;

    void job_bytes(const Device &d, const Job &j, uint64_t *up, uint64_t *down) const;
    void issue_loop(Device &d);
    void complete_loop(Device &d);
    cfb_error issue(Device &d, Slot &s);
};

// PCIe bytes a job moves in either direction (the sparse size is the device's running estimate)
void cfb_pool::job_bytes(const Device &d, const Job &j, uint64_t *up, uint64_t *down) const
{
    const uint64_t coded = j.sparse ? (uint64_t)(d.value_guess ? d.value_guess : layout.coded_bytes / 8) : (uint64_t)layout.coded_bytes;
    const uint64_t frame = (uint64_t)layout.frame_bytes;
    if (!j.inverse) { *up = frame; *down = coded; } else { *up = coded; *down = frame; }
}

// enqueue the three stages of one batch; never waits for the GPU
cfb_error cfb_pool::issue(Device &d, Slot &s)
{
    const int n = (int)s.jobs.size();
    const Job &j0 = *s.jobs[0];
    const void *src[kMaxBatch];
    void *dst[kMaxBatch];
    for (int i = 0; i < n; i++) { src[i] = s.jobs[i]->src; dst[i] = s.jobs[i]->dst; }
    cudaStream_t compute = s.ctx->stream, s_up = d.s_up[s.lane], s_down = d.s_down[s.lane];
    cfb_error e;
    if (!j0.inverse) {
        e = stage_fwd_upload(s.codec, n, src, j0.pitch, s_up);
        if (e) return e;
        CFB_CUDA(cudaEventRecord(s.ev_up, s_up));
        CFB_CUDA(cudaStreamWaitEvent(compute, s.ev_up, 0));
        e = stage_fwd_compute(s.codec, n, &j0.quant, j0.sparse);
        if (e) return e;
        CFB_CUDA(cudaEventRecord(s.ev_k, compute));
        CFB_CUDA(cudaStreamWaitEvent(s_down, s.ev_k, 0));
        s.guess = d.value_guess ? d.value_guess : sparse_initial_guess(s.codec);
        e = stage_fwd_download(s.codec, n, dst, j0.sparse, s.guess, s_down);
        if (e) return e;
    } else {
        e = stage_inv_upload(s.codec, n, src, j0.sparse, s_up);
        if (e) return e;
        CFB_CUDA(cudaEventRecord(s.ev_up, s_up));
        CFB_CUDA(cudaStreamWaitEvent(compute, s.ev_up, 0));
        e = stage_inv_compute(s.codec, n, &j0.quant, j0.out_format, j0.sparse);
        if (e) return e;
        CFB_CUDA(cudaEventRecord(s.ev_k, compute));
        CFB_CUDA(cudaStreamWaitEvent(s_down, s.ev_k, 0));
        e = stage_inv_download(s.codec, n, dst, j0.pitch, j0.out_format, s_down);
        if (e) return e;
    }
    CFB_CUDA(cudaEventRecord(s.ev_down, s_down));
    return CFB_OK;
}

void cfb_pool::issue_loop(Device &d)
{
    cudaSetDevice(d.device);
    cfb_bind_thread_to_device(d.device);            // copies are issued from the GPU's own NUMA node
    for (;;) {
        int si = -1;
        {
            std::unique_lock<std::mutex> lk(mu);
            for (;;) {
                bool have_job = false;
                for (auto &j : queue) if (!j->taken && j->device_index == d.index) { have_job = true; break; }
                if (have_job && !d.free_slots.empty()) break;
                if (stopping && !have_job) { d.issuer_done = true; d.cv_flight.notify_all(); return; }
                cv_work.wait(lk);
            }
            si = d.free_slots.front();
            d.free_slots.pop_front();
            Slot &s = *d.slots[si];
            s.jobs.clear();
            // Direction-balanced issue.  A forward job loads the upload direction (frame up, coefficients down), an
            // inverse job the download direction; issuing strictly in submission order lets runs of one kind fill every
            // slot and idle the other copy engine.  Delivery order is what the contract fixes, not execution order: of
            // the oldest untaken forward job and the oldest untaken inverse job of this GPU, take the one that leaves
            // the two directions' outstanding bytes better balanced (ties and starvation: the older one; a job is never
            // overtaken by more than kMaxOvertake younger ones).
            std::shared_ptr<Job> first[2];
            int age[2] = {0, 0}, seen = 0;
            for (auto &j : queue) {
                if (j->taken || j->device_index != d.index) continue;
                const int kind = j->inverse ? 1 : 0;
                if (!first[kind]) { first[kind] = j; age[kind] = seen; }
                seen++;
                if (first[0] && first[1]) break;
            }
            int pick = first[0] ? 0 : 1;
            if (first[0] && first[1]) {
                uint64_t u0, d0, u1, d1;
                job_bytes(d, *first[0], &u0, &d0);
                job_bytes(d, *first[1], &u1, &d1);
                const uint64_t m0 = std::max(d.up_pending + u0, d.down_pending + d0), m1 = std::max(d.up_pending + u1, d.down_pending + d1);
                const int older = age[0] < age[1] ? 0 : 1;
                pick = (m0 == m1) ? older : (m0 < m1 ? 0 : 1);
                if (pick != older && first[older]->overtaken >= kMaxOvertake) pick = older;
                if (pick != older) first[older]->overtaken++;
            }
            const Job &a = *first[pick];
            // up to `batch` untaken jobs of this device with the same direction, format and quant table
            for (auto &j : queue) {
                if (j->taken || j->device_index != d.index) continue;
                if (j->inverse != a.inverse || j->sparse != a.sparse || j->out_format != a.out_format || j->pitch != a.pitch ||
                    memcmp(&j->quant, &a.quant, sizeof(cfb_quant)) != 0)
                    continue;
                j->taken = true;
                s.jobs.push_back(j);
                if ((int)s.jobs.size() == batch) break;
            }
            s.up_bytes = s.down_bytes = 0;
            for (auto &j : s.jobs) { uint64_t u, dn; job_bytes(d, *j, &u, &dn); s.up_bytes += u; s.down_bytes += dn; }
            d.up_pending += s.up_bytes; d.down_pending += s.down_bytes;
        }
        Slot &s = *d.slots[si];
        s.issue_error = issue(d, s);
        if (s.issue_error != CFB_OK) {
            // whatever was enqueued before the failure must drain before the staging is reused
            cudaStreamSynchronize(d.s_up[s.lane]); cudaStreamSynchronize(s.ctx->stream); cudaStreamSynchronize(d.s_down[s.lane]);
            cudaGetLastError();
        }
        {
            std::lock_guard<std::mutex> lk(mu);
            d.in_flight.push_back(si);
        }
        d.cv_flight.notify_one();
    }
}

void cfb_pool::complete_loop(Device &d)
{
    cudaSetDevice(d.device);
    cfb_bind_thread_to_device(d.device);
    for (;;) {
        int si;
        {
            std::unique_lock<std::mutex> lk(mu);
            d.cv_flight.wait(lk, [&] { return !d.in_flight.empty() || d.issuer_done; });
            if (d.in_flight.empty()) return;        // the issuer has stopped and everything it issued has been delivered
            si = d.in_flight.front();
        }
        Slot &s = *d.slots[si];
        cfb_error e = s.issue_error;
        unsigned maxv = 0;
        if (e == CFB_OK) {
            const cudaError_t ce = cudaEventSynchronize(s.ev_down);
            if (ce != cudaSuccess) e = cuda_fail(ce, "cudaEventSynchronize(download)");
        }
        if (e == CFB_OK && !s.jobs[0]->inverse && s.jobs[0]->sparse) {
            const int n = (int)s.jobs.size();
            void *dst[kMaxBatch];
            for (int i = 0; i < n; i++) dst[i] = s.jobs[i]->dst;
            bool more = false;
            e = stage_fwd_tail(s.codec, n, dst, s.guess, d.s_down[s.lane], nullptr, &maxv, &more);
            if (e == CFB_OK && more) {
                const cudaError_t ce = cudaStreamSynchronize(d.s_down[s.lane]);
                if (ce != cudaSuccess) e = cuda_fail(ce, "cudaStreamSynchronize(download tail)");
            }
        }
        {
            std::lock_guard<std::mutex> lk(mu);
            if (maxv) d.value_guess = sparse_next_guess(s.codec, maxv);
            for (auto &j : s.jobs) { j->error = e; j->done = true; }
            s.jobs.clear();
            d.up_pending -= s.up_bytes; d.down_pending -= s.down_bytes;
            d.in_flight.pop_front();
            d.free_slots.push_back(si);
        }
        cv_done.notify_all();
        cv_work.notify_all();       // a slot is free again
    }
}

extern "C" {

cfb_error cfb_host_alloc(size_t bytes, void **out)
{
    if (!out) return CFB_ERROR_INVALID_ARGUMENT;
    *out = nullptr;
    CFB_CUDA(cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocPortable));
    return CFB_OK;
}

void cfb_host_free(void *p) { if (p) cudaFreeHost(p); }

static void destroy_device(Device &d)
{
    cudaSetDevice(d.device);
    for (auto &s : d.slots) {
        if (s->codec) cfb_codec_destroy(s->codec);
        if (s->ctx) cfb_context_destroy(s->ctx);
        if (s->ev_up) cudaEventDestroy(s->ev_up);
        if (s->ev_k) cudaEventDestroy(s->ev_k);
        if (s->ev_down) cudaEventDestroy(s->ev_down);
    }
    for (int k = 0; k < kCopyStreams; k++) {
        if (d.s_up[k]) cudaStreamDestroy(d.s_up[k]);
        if (d.s_down[k]) cudaStreamDestroy(d.s_down[k]);
    }
}

cfb_error cfb_pool_create(const int *devices, int ndevices, const cfb_frame_desc *desc,
                          int slots, int batch, int queue_length, cfb_pool **out)
{
    if (!devices || !desc || !out || ndevices < 1) { set_error("null/empty argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    *out = nullptr;
    if (slots < 1 || slots > 32 || batch < 1 || batch > CFB_MAX_BATCH || queue_length < 1) {
        set_error("slots %d (1..32), batch %d (1..%d), queue_length %d (>=1) out of range", slots, batch, CFB_MAX_BATCH, queue_length);
        return CFB_ERROR_INVALID_ARGUMENT;
    }
    cfb_layout lay;
    cfb_error err = cfb_layout_compute(desc, &lay);
    if (err) return err;
    std::unique_ptr<cfb_pool> p(new (std::nothrow) cfb_pool());
    if (!p) return CFB_ERROR_OUTOFMEMORY;
    p->desc = *desc; p->layout = lay; p->batch = batch; p->queue_length = queue_length;
    p->devices.assign(devices, devices + ndevices);
    for (int di = 0; di < ndevices && !err; di++) {
        std::unique_ptr<Device> d(new Device());
        d->device = devices[di]; d->index = di;
        {
            cudaError_t ce = cudaSetDevice(devices[di]);
            for (int k = 0; k < kCopyStreams && ce == cudaSuccess; k++) {
                ce = cudaStreamCreateWithFlags(&d->s_up[k], cudaStreamNonBlocking);
                if (ce == cudaSuccess) ce = cudaStreamCreateWithFlags(&d->s_down[k], cudaStreamNonBlocking);
            }
            if (ce != cudaSuccess) err = cuda_fail(ce, "cudaStreamCreate(pool copy streams)");
        }
        for (int k = 0; k < slots && !err; k++) {
            std::unique_ptr<Slot> s(new Slot());
            s->lane = k % kCopyStreams;
            err = cfb_context_create(devices[di], &s->ctx);
            if (!err) err = cfb_codec_create(s->ctx, desc, batch, &s->codec);
            if (!err) {
                cudaError_t ce = cudaEventCreateWithFlags(&s->ev_up, cudaEventDisableTiming);
                if (ce == cudaSuccess) ce = cudaEventCreateWithFlags(&s->ev_k, cudaEventDisableTiming);
                if (ce == cudaSuccess) ce = cudaEventCreateWithFlags(&s->ev_down, cudaEventBlockingSync | cudaEventDisableTiming);
                if (ce != cudaSuccess) err = cuda_fail(ce, "cudaEventCreate(pool)");
            }
            d->free_slots.push_back((int)d->slots.size());
            d->slots.push_back(std::move(s));
        }
        p->devs.push_back(std::move(d));
    }
    if (err) {
        for (auto &d : p->devs) destroy_device(*d);
        return err;
    }
    cfb_pool *raw = p.release();
    for (auto &d : raw->devs) {
        d->issuer = std::thread(&cfb_pool::issue_loop, raw, std::ref(*d));
        d->completer = std::thread(&cfb_pool::complete_loop, raw, std::ref(*d));
    }
    *out = raw;
    return CFB_OK;
}

cfb_error cfb_pool_set_interlaced(cfb_pool *pool, int interlaced)
{
    if (!pool) { set_error("null pool"); return CFB_ERROR_INVALID_ARGUMENT; }
    std::lock_guard<std::mutex> lk(pool->mu);          // applies to jobs submitted after this call returns
    for (auto &d : pool->devs)
        for (auto &s : d->slots) {
            cfb_error e = cfb_codec_set_interlaced(s->codec, interlaced);
            if (e) return e;
        }
    return CFB_OK;
}

cfb_error cfb_pool_set_decode_resolution(cfb_pool *pool, int resolution)
{
    if (!pool) { set_error("null pool"); return CFB_ERROR_INVALID_ARGUMENT; }
    std::lock_guard<std::mutex> lk(pool->mu);          // applies to jobs submitted after this call returns
    for (auto &d : pool->devs)
        for (auto &s : d->slots) {
            cfb_error e = cfb_codec_set_decode_resolution(s->codec, resolution);
            if (e) return e;
        }
    return CFB_OK;
}

cfb_error cfb_pool_set_bayer_phase(cfb_pool *pool, int bayer_format)
{
    if (!pool) { set_error("null pool"); return CFB_ERROR_INVALID_ARGUMENT; }
    std::lock_guard<std::mutex> lk(pool->mu);          // applies to jobs submitted after this call returns
    for (auto &d : pool->devs)
        for (auto &s : d->slots) {
            cfb_error e = cfb_codec_set_bayer_phase(s->codec, bayer_format);
            if (e) return e;
        }
    return CFB_OK;
}

cfb_error cfb_pool_set_bayer_curve(cfb_pool *pool, const uint16_t *curve, int entries)
{
    if (!pool) { set_error("null pool"); return CFB_ERROR_INVALID_ARGUMENT; }
    std::lock_guard<std::mutex> lk(pool->mu);          // applies to jobs submitted after this call returns
    for (auto &d : pool->devs)
        for (auto &s : d->slots) {
            cfb_error e = cfb_codec_set_bayer_curve(s->codec, curve, entries);
            if (e) return e;
        }
    return CFB_OK;
}

cfb_error cfb_pool_set_bayer_decode_curve(cfb_pool *pool, const uint16_t *table, int entries)
{
    if (!pool) { set_error("null pool"); return CFB_ERROR_INVALID_ARGUMENT; }
    std::lock_guard<std::mutex> lk(pool->mu);          // applies to jobs submitted after this call returns
    for (auto &d : pool->devs)
        for (auto &s : d->slots) {
            cfb_error e = cfb_codec_set_bayer_decode_curve(s->codec, table, entries);
            if (e) return e;
        }
    return CFB_OK;
}

void cfb_pool_destroy(cfb_pool *pool)
{
    if (!pool) return;
    {
        std::lock_guard<std::mutex> lk(pool->mu);
        pool->stopping = true;
    }
    pool->cv_work.notify_all();
    for (auto &d : pool->devs) if (d->issuer.joinable()) d->issuer.join();      // issues whatever is still queued
    for (auto &d : pool->devs) if (d->completer.joinable()) d->completer.join();
    for (auto &d : pool->devs) destroy_device(*d);
    delete pool;
}

static cfb_error pool_submit(cfb_pool *pool, std::shared_ptr<Job> job)
{
    {
        std::unique_lock<std::mutex> lk(pool->mu);
        pool->cv_space.wait(lk, [&] { return (int)pool->queue.size() < pool->queue_length; });
        job->device_index = (int)(pool->submitted % pool->devices.size());     // EncoderPool.cpp:284
        pool->submitted++;
        pool->queue.push_back(std::move(job));
    }
    pool->cv_work.notify_all();
    return CFB_OK;
}

cfb_error cfb_pool_submit_forward(cfb_pool *pool, uint32_t frame_number, const void *h_frame, int frame_pitch,
                                  const cfb_quant *quant, void *h_coded)
{
    if (!pool || !h_frame || !quant || !h_coded) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    auto j = std::make_shared<Job>();
    j->frame_number = frame_number; j->inverse = false; j->src = h_frame; j->dst = h_coded; j->pitch = frame_pitch; j->quant = *quant;
    return pool_submit(pool, std::move(j));
}

cfb_error cfb_pool_submit_inverse(cfb_pool *pool, uint32_t frame_number, const void *h_coded,
                                  const cfb_quant *quant, int out_format, void *h_frame, int frame_pitch)
{
    if (!pool || !h_frame || !quant || !h_coded) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    auto j = std::make_shared<Job>();
    j->frame_number = frame_number; j->inverse = true; j->src = h_coded; j->dst = h_frame; j->pitch = frame_pitch;
    j->out_format = out_format; j->quant = *quant;
    return pool_submit(pool, std::move(j));
}

cfb_error cfb_pool_submit_forward_sparse(cfb_pool *pool, uint32_t frame_number, const void *h_frame, int frame_pitch,
                                         const cfb_quant *quant, void *h_sparse)
{
    if (!pool || !h_frame || !quant || !h_sparse) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    auto j = std::make_shared<Job>();
    j->frame_number = frame_number; j->inverse = false; j->sparse = true; j->src = h_frame; j->dst = h_sparse; j->pitch = frame_pitch; j->quant = *quant;
    return pool_submit(pool, std::move(j));
}

cfb_error cfb_pool_submit_inverse_sparse(cfb_pool *pool, uint32_t frame_number, const void *h_sparse,
                                         const cfb_quant *quant, int out_format, void *h_frame, int frame_pitch)
{
    if (!pool || !h_frame || !quant || !h_sparse) { set_error("null argument"); return CFB_ERROR_INVALID_ARGUMENT; }
    auto j = std::make_shared<Job>();
    j->frame_number = frame_number; j->inverse = true; j->sparse = true; j->src = h_sparse; j->dst = h_frame; j->pitch = frame_pitch;
    j->out_format = out_format; j->quant = *quant;
    return pool_submit(pool, std::move(j));
}

static cfb_error pool_pop(cfb_pool *pool, bool block, uint32_t *frame_number, cfb_error *job_error)
{
    if (!pool) return CFB_ERROR_INVALID_ARGUMENT;
    std::shared_ptr<Job> j;
    {
        std::unique_lock<std::mutex> lk(pool->mu);
        if (pool->queue.empty()) { set_error("no job outstanding"); return CFB_ERROR_INVALID_ARGUMENT; }
        if (!pool->queue.front()->done) {
            if (!block) return CFB_ERROR_NOT_FINISHED;
            pool->cv_done.wait(lk, [&] { return pool->queue.front()->done; });
        }
        j = pool->queue.front();
        pool->queue.pop_front();
    }
    pool->cv_space.notify_all();
    if (frame_number) *frame_number = j->frame_number;
    if (job_error) *job_error = j->error;
    return CFB_OK;
}

cfb_error cfb_pool_wait(cfb_pool *pool, uint32_t *frame_number, cfb_error *job_error) { return pool_pop(pool, true, frame_number, job_error); }
cfb_error cfb_pool_test(cfb_pool *pool, uint32_t *frame_number, cfb_error *job_error) { return pool_pop(pool, false, frame_number, job_error); }

cfb_error cfb_pool_stats(cfb_pool *pool, cfb_stats *out)
{
    if (!pool || !out) return CFB_ERROR_INVALID_ARGUMENT;
    memset(out, 0, sizeof(*out));
    for (auto &d : pool->devs)
        for (auto &s : d->slots) {
            cfb_stats t;
            cfb_context_stats(s->ctx, &t);
            out->kernel_launches += t.kernel_launches; out->frames_forward += t.frames_forward; out->frames_inverse += t.frames_inverse;
            out->h2d_bytes += t.h2d_bytes; out->d2h_bytes += t.d2h_bytes;
        }
    return CFB_OK;
}

}  // extern "C"
