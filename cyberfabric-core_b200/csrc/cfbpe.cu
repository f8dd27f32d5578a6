// cfbpe.cu -- libcfbpe.so: device context, vocab upload and the C ABI of include/cfbpe.h.
//
// Built for sm_90a (H100) only.  There is no CPU path in this library: every entry point that
// computes runs the kernels of bpe_kernels.cuh on the device or returns an error.
#include <cuda_runtime.h>

#include <array>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/cfbpe.h"

struct ProfEvents;
#define CFBPE_LAUNCH(kernel, grid, block, stream, ...) kernel<<<(grid), (block), 0, (stream)>>>(__VA_ARGS__)
#define CFBPE_LAUNCH_SMEM(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#define CFBPE_ZERO(ptr, bytes, stream) cudaMemsetAsync((ptr), 0, (bytes), (stream))
#define CFBPE_MARK(prof, idx, stream, begin) prof_mark((prof), (idx), (stream), (begin))
static inline void prof_mark(ProfEvents* p, int idx, cudaStream_t s, bool begin);
// make `aux` wait for what is queued on `main` so far / make `main` wait for `aux`; no-ops when both are the same stream
#define CFBPE_FORK(main, aux, ev) do { if ((main) != (aux)) { cudaEventRecord((ev), (main)); cudaStreamWaitEvent((aux), (ev), 0); } } while (0)
#define CFBPE_JOIN(main, aux, ev) do { if ((main) != (aux)) { cudaEventRecord((ev), (aux)); cudaStreamWaitEvent((main), (ev), 0); } } while (0)

#include "pipeline.cuh"
#include "pretok_ctx.h"
#include "specials.cuh"
#include "subbatch.h"
#include "unicode_tables.h"
#include "utf8_repair.cuh"
#include "vocab.h"

using namespace cfbpe;

// Owners of a context's CUDA resources.  Each kind is released by its deleter and nowhere else; a deleter acts on the current
// device, so ~Lane and ~DeviceCtx select theirs before their members go.
struct DeviceFree { void operator()(void* p) const { cudaFree(p); } };
struct HostFree { void operator()(void* p) const { cudaFreeHost(p); } };
struct StreamDestroy { void operator()(cudaStream_t s) const { cudaStreamDestroy(s); } };
struct EventDestroy { void operator()(cudaEvent_t e) const { cudaEventDestroy(e); } };
template <typename T> using DevPtr = std::unique_ptr<T, DeviceFree>;    // device memory
template <typename T> using HostPtr = std::unique_ptr<T, HostFree>;     // pinned host memory
using Stream = std::unique_ptr<std::remove_pointer_t<cudaStream_t>, StreamDestroy>;
using Event = std::unique_ptr<std::remove_pointer_t<cudaEvent_t>, EventDestroy>;

struct ProfEvents {
    Event ev[CFBPE_NUM_KERNELS][2];
    Event h2d[2], d2h[2], total[2];
    bool launched[CFBPE_NUM_KERNELS];
};
static inline void prof_mark(ProfEvents* p, int idx, cudaStream_t s, bool begin) {
    if (!p) return;
    cudaEventRecord(p->ev[idx][begin ? 0 : 1].get(), s);
    p->launched[idx] = true;
}

#include <dlfcn.h>

#include <atomic>
#include <shared_mutex>
#include <thread>

constexpr int kMaxPipeChunks = 64;
constexpr int kSideStreams = 16;
constexpr int kPrioLevels = 8, kPoolSlots = 9;
constexpr int kTracePoints = 8;     // CFBPE_PIPE_TRACE: events per sub-batch
#ifndef CFBPE_FRONT_STREAMS
#define CFBPE_FRONT_STREAMS 6
#endif
constexpr int kFrontStreams = CFBPE_FRONT_STREAMS;
constexpr uint64_t kPipeChunkBytes = 12ull << 20;   // largest sub-batch of a pipelined host call (the sizes ramp up to it and down again); on H100 8, 16 and 24 MB are within the noise of it
constexpr uint64_t kPipeMinBytes = 4ull << 20;      // smaller calls run as one shot (a 134 MB batch sharded over 8 GPUs is 16.8 MB a rank: it must still pipeline)

// ---------------------------------------------------------------------------------------
// Structure of a context (SURVEY.md section 8(b): "cfbpe_create(cfg: devices[], n_devices, ...)", "safe to call concurrently from
// several host threads (internal stream pool ...)"):
//   cfbpe_ctx  ->  one DeviceCtx per CUDA device (its copy of every vocabulary's tables, its NCCL communicator)
//              ->  n_workspaces Lanes per device: a Lane is everything ONE call touches on the device -- streams, events, the
//                  workspace, staging buffers, pinned status words -- so calls on different lanes run concurrently.
// A call takes a lane (try-lock round robin, else it waits for one), holds the vocabularies shared (vocab_load holds them
// exclusively) and sets no state outside its lane; the last error is per THREAD.
// A multi-device context shards a host batch by bytes on prompt boundaries, one host thread per device; NCCL (dlopen'ed
// libnccl.so.2: the library links no NCCL symbol) broadcasts the packed tables at vocab load and all-gathers the per-shard
// token totals of every batch, from which each device rebases its offsets (SURVEY.md section 8(e)).
// ---------------------------------------------------------------------------------------
// the buffers of special-token calls (cfbpe_encode_batch_special*), allocated on the lane's first such call: a context that
// never uses special tokens keeps the footprint it had
struct LaneSpecial {
    DevPtr<uint32_t> kept_n;              // [max_prompts] kept matches per prompt ...
    DevPtr<uint64_t> kept_base;           // ... and their exclusive scan
    DevPtr<uint64_t> st_off;              // [max_prompts + 1] stretch byte offsets
    DevPtr<uint8_t> st_vocab;             // [max_prompts] stretch vocabularies
    DevPtr<uint32_t> st_id;               // [max_prompts] special id of a stretch, or kSpText
    DevPtr<uint64_t> st_base;             // [max_prompts] first output id of a stretch
    DevPtr<uint64_t> fin_offsets;         // host calls: the prompts' offsets [max_prompts + 1] ...
    DevPtr<uint32_t> fin_counts;          // ... and counts [max_prompts]
    DevPtr<uint8_t> modes;                // [CFBPE_MAX_VOCABS][kMaxSpecials] the call's mode bytes
    DevPtr<SpecialStatus> status;
    HostPtr<SpecialStatus> h_status;      // pinned
};

// the buffers of lossy calls (cfbpe_encode_batch_lossy*), allocated on the lane's first such call, all or none: a context that never
// makes one keeps the footprint it had
struct LaneLossy {
    DevPtr<uint64_t> offsets;             // [max_prompts + 1] the prompts' offsets in the repaired batch
    DevPtr<uint32_t> replaced;            // [max_prompts] U+FFFD inserted per prompt
    DevPtr<LossyStatus> status;
    HostPtr<LossyStatus> h_status;        // pinned
};

struct Lane {
    std::mutex mu;                        // held for the duration of a call
    int device = 0;
    uint64_t max_bytes = 0;
    Stream stream;                       // compute
    Stream h2d_stream;                   // pipelined host calls: uploads run ahead of the kernels ...
    Stream d2h_stream;                   // ... and downloads trail them
    DevPtr<uint32_t> d_dec_sums;         // decode: bytes per tile of kDecodeTile tokens ...
    DevPtr<uint64_t> d_dec_base;         // ... and their exclusive scan
    Stream aux_stream;                   // the long-piece kernel runs here, next to the short-piece kernel
    Stream aux2_stream;                  // ... and the big-piece kernel here, next to both
    Event ev_fork, ev_join, ev_join2;
    Stream side2[kSideStreams];          // pipelined host calls: the big-piece kernel of sub-batch k
    Event ev_list[kMaxPipeChunks];
    Event ev_ws;                         // recorded at the end of an asynchronous device-path call: the workspace is busy until then
    bool ws_pending = false;             // ... and whether one is outstanding
    uint64_t dev_out_cap = 0;            // out_cap of the last device-path call (cfbpe_device_status reports ENOSPC against it)
    bool dev_want_ids = false;
    Event ev_scan[kMaxPipeChunks];
    Stream front[kFrontStreams];         // front streams 1.. of a pipelined host call (0 = stream)
    Stream pool[kPrioLevels][kPoolSlots];   // CFBPE_PIPE_PRIO=1|2 (experiment): streams by priority level
    int prio_mode = 0, prio_levels = 1;
    Stream side[kSideStreams];           // long-piece tails + emit of sub-batch k overlap the front of k+1
    Event ev_front[kMaxPipeChunks];
    Event ev_h2d[kMaxPipeChunks];
    Event ev_done[kMaxPipeChunks];
    Event ev_chain[kMaxPipeChunks];      // tile_scan of sub-batch k done: the next sub-batch's scan may read tok_end
    std::vector<std::array<Event, kTracePoints>> trace;   // CFBPE_PIPE_TRACE=1: timed events per sub-batch (h2d, split, short, long, back, d2h) + [nc][0] = start
    DevPtr<DeviceStatus> d_status_arr;   // one status per sub-batch
    HostPtr<DeviceStatus> h_status_arr;  // pinned
    HostPtr<uint64_t> h_offs_stage;      // pinned: sub-batch-local offsets
    HostPtr<uint64_t> h_totals;          // pinned: the all-gathered token totals of a multi-device call [CFBPE_MAX_DEVICES]
    DevPtr<uint64_t> d_totals;           // device: the same
    // inputs / outputs of the host API
    DevPtr<uint8_t> d_bytes;
    DevPtr<uint64_t> d_offsets;
    DevPtr<uint8_t> d_vocab_ids;
    DevPtr<uint32_t> d_out_ids;
    DevPtr<uint64_t> d_out_offsets;
    DevPtr<uint32_t> d_out_counts;
    DevPtr<uint32_t> d_out_starts;       // host calls with token starts: [max_bytes + 1], allocated on the lane's first such call
    DevPtr<uint32_t> d_trunc;            // host truncate calls: budgets, cuts, kept counts [3 x (max_prompts + 1)], allocated on the
                                         // lane's first such call
    DevPtr<uint32_t> d_unit_lens;        // host unit-start calls with lengths: every prompt's length in units [max_prompts], allocated
                                         // on the lane's first such call
    DevPtr<uint64_t> d_chunk_offs;       // host chunk calls: chunk offsets in the layout of d_out_offsets, then the shard chunk totals
                                         // of a multi-device call [CFBPE_MAX_DEVICES]; allocated on the lane's first such call
    Workspace ws{};                      // the kernels' view: its sized buffers are released by ~Lane, its status is d_status
    DevPtr<DeviceStatus> d_status;
    HostPtr<DeviceStatus> h_status;      // pinned
    ProfEvents prof{};
    LaneSpecial sp;
    LaneLossy lossy;

    ~Lane() {                            // the members' deleters run after this body, on the lane's device
        cudaSetDevice(device);
        for_each_ws_buffer(ws, [](auto*& p, WsKind) { cudaFree(p); });
    }
};

struct DeviceVocab { DevPtr<uint8_t> d_blob; };

struct DeviceCtx {
    int device = 0;
    int index = 0;                        // position in cfbpe_ctx::devs (= NCCL rank)
    int sm_count = 0;                     // set from the device's properties; 0 until then
    DevPtr<uint8_t> d_uc1;
    DevPtr<uint8_t> d_uc2;
    DevPtr<uint8_t> d_ascii;
    DevPtr<uint16_t> d_fsm;
    DevPtr<uint8_t> d_split_tables;      // SplitTablesHost: class bytes, 16-wide transition tables, context + product automata (pretok_ctx.h)
    UcTables uc{};
    DeviceVocab vocabs[CFBPE_MAX_VOCABS];
    VocabSet vs{};
    DevPtr<uint32_t> d_specials[CFBPE_MAX_VOCABS];   // each vocabulary's special-token table (specials.h), or empty
    SpecialSet specials{};                          // their views (modes NULL): what decode reads
    std::vector<std::unique_ptr<Lane>> lanes;
    std::atomic<uint32_t> next_lane{0};
    void* comm = nullptr;                 // ncclComm_t of this device in the context's communicator

    ~DeviceCtx() { cudaSetDevice(device); }   // the members' deleters run after this body, on this device
};

struct HostVocab { bool loaded = false; std::vector<uint8_t> h_blob; TablesHeader hdr{}; };

// the few NCCL entry points the library uses, resolved at cfbpe_create of a multi-device context
struct NcclApi {
    void* lib = nullptr;
    int (*CommInitAll)(void**, int, const int*) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    int (*Broadcast)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};
constexpr int kNcclChar = 0, kNcclUint64 = 5;       // ncclDataType_t values (nccl.h: ncclInt8 = ncclChar = 0, ncclUint64 = 5)

struct cfbpe_ctx {
    std::vector<std::unique_ptr<DeviceCtx>> devs;
    std::shared_mutex vocab_mu;           // calls: shared; vocabulary load / import: exclusive
    HostVocab vocabs[CFBPE_MAX_VOCABS];
    std::vector<uint32_t> specials[CFBPE_MAX_VOCABS];   // the special-token tables (host copies; empty = none registered)
    uint32_t loaded_mask = 0;
    uint64_t max_bytes = 0;
    uint32_t max_prompts = 0;
    uint32_t n_workspaces = 1;
    uint64_t pipe_chunk = kPipeChunkBytes, pipe_min = kPipeMinBytes;   // CFBPE_PIPE_CHUNK_BYTES / CFBPE_PIPE_MIN_BYTES override (tests)
    std::atomic<bool> profiling{false};
    NcclApi nccl;
    bool peer_ok = false;      // several devices, each maps the memory of all the others (NVLink): sub-batches may go round-robin
};

namespace {

// the last error and the last profile are per calling thread: calls run concurrently on one context
thread_local std::string tl_err;
thread_local cfbpe_profile tl_profile{};
thread_local bool tl_profile_ready = false;
thread_local Lane* tl_device_lane = nullptr;      // the lane of this thread's last device-path call (cfbpe_device_status)

int fail(cfbpe_ctx*, int code, const std::string& msg) {
    tl_err = msg;
    return code;
}
#define CK(call)                                                                                         \
    do {                                                                                                 \
        cudaError_t e_ = (call);                                                                         \
        if (e_ != cudaSuccess) {                                                                         \
            return fail(ctx, CFBPE_EIO, std::string(#call) + ": " + cudaGetErrorString(e_));             \
        }                                                                                                \
    } while (0)

template <typename T>
cudaError_t dmalloc(T** p, uint64_t count) { return cudaMalloc(reinterpret_cast<void**>(p), count * sizeof(T)); }
// fill an owner: count elements of T on the current device (dmalloc) or in pinned host memory (hmalloc), a stream, an event; the
// owner stays empty when the call fails
template <typename T>
cudaError_t dmalloc(DevPtr<T>& p, uint64_t count) {
    T* raw = nullptr;
    const cudaError_t e = dmalloc(&raw, count);
    p.reset(e == cudaSuccess ? raw : nullptr);
    return e;
}
template <typename T>
cudaError_t hmalloc(HostPtr<T>& p, uint64_t count) {
    void* raw = nullptr;
    const cudaError_t e = cudaMallocHost(&raw, count * sizeof(T));
    p.reset(e == cudaSuccess ? static_cast<T*>(raw) : nullptr);
    return e;
}
cudaError_t make_stream(Stream& s, int priority) {
    cudaStream_t raw = nullptr;
    const cudaError_t e = cudaStreamCreateWithPriority(&raw, cudaStreamNonBlocking, priority);
    s.reset(e == cudaSuccess ? raw : nullptr);
    return e;
}
cudaError_t make_event(Event& ev, unsigned flags) {
    cudaEvent_t raw = nullptr;
    const cudaError_t e = cudaEventCreateWithFlags(&raw, flags);
    ev.reset(e == cudaSuccess ? raw : nullptr);
    return e;
}

// the error a pass's status reports (status_error), or CFBPE_OK
int fail_status(cfbpe_ctx* ctx, const DeviceStatus& st) {
    const StatusError e = status_error(st);
    return e.code ? fail(ctx, e.code, e.msg) : CFBPE_OK;
}
// out_cap is too small for the call's `need` ids; a host call also learns it in out_offsets[n]
int fail_nospace(cfbpe_ctx* ctx, uint64_t need, uint64_t* out_offsets = nullptr, uint32_t n = 0) {
    if (out_offsets) out_offsets[n] = need;
    return fail(ctx, CFBPE_ENOSPC, "out_cap too small: need " + std::to_string(need) + " ids");
}

// a free lane of the device, locked: round robin without waiting; when all are busy, wait for the next in turn
struct LaneLock {
    Lane* ln = nullptr;
    explicit LaneLock(DeviceCtx* dv) {
        const uint32_t n = static_cast<uint32_t>(dv->lanes.size()), start = dv->next_lane.fetch_add(1);
        for (uint32_t i = 0; i < n && !ln; ++i) { Lane* c = dv->lanes[(start + i) % n].get(); if (c->mu.try_lock()) ln = c; }
        if (!ln) { ln = dv->lanes[start % n].get(); ln->mu.lock(); }
    }
    ~LaneLock() { if (ln) ln->mu.unlock(); }
    LaneLock(const LaneLock&) = delete;
    LaneLock& operator=(const LaneLock&) = delete;
};

int validate_batch(cfbpe_ctx* ctx, uint32_t n, const uint64_t* offsets, const uint8_t* vocab_ids, uint64_t* total_out) {
    if (n > ctx->max_prompts) return fail(ctx, CFBPE_EINVAL, "n_prompts exceeds max_prompts of this context");
    if (!offsets) return fail(ctx, CFBPE_EINVAL, "offsets is NULL");
    if (offsets[0] != 0) return fail(ctx, CFBPE_EINVAL, "offsets[0] must be 0");
    for (uint32_t i = 0; i < n; ++i)
        if (offsets[i + 1] < offsets[i]) return fail(ctx, CFBPE_EINVAL, "offsets are not monotonic at prompt " + std::to_string(i));
    if (offsets[n] > ctx->max_bytes * ctx->devs.size()) return fail(ctx, CFBPE_EINVAL, "batch exceeds max_batch_bytes of this context");
    if (vocab_ids) {
        for (uint32_t i = 0; i < n; ++i)
            if (vocab_ids[i] >= CFBPE_MAX_VOCABS || !ctx->vocabs[vocab_ids[i]].loaded)
                return fail(ctx, CFBPE_ENOENT, "prompt " + std::to_string(i) + " names a vocab that is not loaded");
    } else if (!ctx->vocabs[0].loaded) {
        return fail(ctx, CFBPE_ENOENT, "vocab 0 is not loaded");
    }
    *total_out = offsets[n];
    return CFBPE_OK;
}

// Drop the special-token table of a vocabulary on every device (caller holds vocab_mu exclusively)
void clear_specials(cfbpe_ctx* ctx, uint32_t vocab_id) {
    ctx->specials[vocab_id].clear();
    for (auto& dvp : ctx->devs) {
        DeviceCtx* dv = dvp.get();
        dv->specials.v[vocab_id] = SpecialView{};
        if (dv->d_specials[vocab_id]) {
            cudaSetDevice(dv->device);
            cudaDeviceSynchronize();          // a device-path call may still read the table
            dv->d_specials[vocab_id].reset();
        }
    }
}

// Install a packed table blob as vocabulary vocab_id on EVERY device of the context (caller holds vocab_mu exclusively).
// Device 0 gets it from the host; with several devices the others get it from device 0 by ncclBroadcast over NVLink -- the rank
// file was parsed once, the tables crossed PCIe once.
int install_blob(cfbpe_ctx* ctx, uint32_t vocab_id, std::vector<uint8_t>&& blob) {
    const size_t G = ctx->devs.size();
    std::vector<DevPtr<uint8_t>> nb(G);      // the new tables, one a device: released on return unless installed
    for (size_t d = 0; d < G; ++d) {
        cudaSetDevice(ctx->devs[d]->device);
        if (dmalloc(nb[d], blob.size()) != cudaSuccess) {
            cudaGetLastError();
            return fail(ctx, CFBPE_ENOMEM, "no device memory for the vocabulary tables");
        }
    }
    cudaSetDevice(ctx->devs[0]->device);
    cudaError_t e = cudaMemcpy(nb[0].get(), blob.data(), blob.size(), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) return fail(ctx, CFBPE_EIO, std::string("table upload: ") + cudaGetErrorString(e));
    if (G > 1) {
        const NcclApi& nc = ctx->nccl;
        int rc = nc.GroupStart();
        for (size_t d = 0; d < G && rc == 0; ++d) {
            cudaSetDevice(ctx->devs[d]->device);
            cudaStream_t st = ctx->devs[d]->lanes[0]->stream.get();
            rc = nc.Broadcast(nb[0].get(), nb[d].get(), blob.size(), kNcclChar, 0, ctx->devs[d]->comm, st);
        }
        const int rc2 = nc.GroupEnd();
        if (rc == 0) rc = rc2;
        for (size_t d = 0; d < G; ++d) { cudaSetDevice(ctx->devs[d]->device); if (cudaStreamSynchronize(ctx->devs[d]->lanes[0]->stream.get()) != cudaSuccess && rc == 0) rc = -1; }
        if (rc != 0) return fail(ctx, CFBPE_EIO, std::string("ncclBroadcast of the vocabulary tables: ") + (rc > 0 ? nc.GetErrorString(rc) : "stream error"));
    }
    clear_specials(ctx, vocab_id);           // a new vocabulary starts without special tokens
    HostVocab& hv = ctx->vocabs[vocab_id];
    hv.h_blob = std::move(blob);
    std::memcpy(&hv.hdr, hv.h_blob.data(), sizeof(TablesHeader));
    hv.loaded = true;
    ctx->loaded_mask |= 1u << vocab_id;
    for (size_t d = 0; d < G; ++d) {
        DeviceCtx* dv = ctx->devs[d].get();
        cudaSetDevice(dv->device);
        DeviceVocab& v = dv->vocabs[vocab_id];
        if (v.d_blob) cudaDeviceSynchronize();   // kernels of a device-path call on any stream may still read the old tables
        v.d_blob = std::move(nb[d]);
        dv->vs.v[vocab_id] = make_view(v.d_blob.get(), hv.hdr);
        dv->vs.loaded_mask = ctx->loaded_mask;
        // slots that are not loaded alias a loaded one: a bad vocabulary id handed in by a device-path caller is reported
        // (DeviceStatus::bad_vocab -> CFBPE_ENOENT) instead of dereferencing a null table
        for (uint32_t i = 0; i < CFBPE_MAX_VOCABS; ++i) if (!ctx->vocabs[i].loaded) dv->vs.v[i] = dv->vs.v[vocab_id];
    }
    return CFBPE_OK;
}

void fill_profile(Lane* ln, uint64_t n_bytes) {
    cfbpe_profile& p = tl_profile;
    std::memset(&p, 0, sizeof p);
    for (int k = 0; k < CFBPE_NUM_KERNELS; ++k) {
        if (!ln->prof.launched[k]) continue;
        float ms = 0;
        if (cudaEventElapsedTime(&ms, ln->prof.ev[k][0].get(), ln->prof.ev[k][1].get()) == cudaSuccess) p.kernel_ms[k] = ms;
        p.kernel_launches[k] = (k == K_EMIT) ? 2 : 1;   // emit_compact + prompt_offsets
    }
    float ms = 0;
    if (cudaEventElapsedTime(&ms, ln->prof.h2d[0].get(), ln->prof.h2d[1].get()) == cudaSuccess) p.h2d_ms = ms;
    if (cudaEventElapsedTime(&ms, ln->prof.d2h[0].get(), ln->prof.d2h[1].get()) == cudaSuccess) p.d2h_ms = ms;
    if (cudaEventElapsedTime(&ms, ln->prof.total[0].get(), ln->prof.total[1].get()) == cudaSuccess) p.total_ms = ms;
    p.n_tokens = ln->h_status->n_tokens;
    p.n_long_pieces = static_cast<uint64_t>(ln->h_status->n_long) + ln->h_status->n_big;
    p.n_bytes = n_bytes;
    p.n_long_bytes = ln->h_status->long_bytes;
    p.n_long_tokens = ln->h_status->long_tokens;
    p.n_miss_pieces = static_cast<uint64_t>(ln->h_status->miss_n[0]) + ln->h_status->miss_n[1] + ln->h_status->miss_n[2];
    p.n_list_pieces = ln->h_status->defer_n;
    p.n_list_parts = ln->h_status->defer_parts;
    p.n_extra_tokens = ln->h_status->extra_n;
    tl_profile_ready = true;
}

// A lane buffer that only some calls use, allocated on the lane's first such call: a context that never makes one keeps the
// footprint it had.  The caller has selected the lane's device.
template <typename T>
int ensure_lane_buffer(cfbpe_ctx* ctx, DevPtr<T>& p, uint64_t count, const char* what) {
    if (p || dmalloc(p, count) == cudaSuccess) return CFBPE_OK;
    cudaGetLastError();
    return fail(ctx, CFBPE_ENOMEM, std::string("no device memory for ") + what);
}
// the lane buffers of a call with token starts (cfbpe_encode_batch_starts, chunk calls), of a truncate call, of a host chunk call,
// of a host unit-start call with lengths
int ensure_call_buffers(cfbpe_ctx* ctx, Lane* ln, bool starts, bool trunc, bool chunk, bool lens = false) {
    const uint64_t mp = ctx->max_prompts;
    int rc = starts ? ensure_lane_buffer(ctx, ln->d_out_starts, ln->max_bytes + 1, "the token starts") : CFBPE_OK;
    if (!rc && trunc) rc = ensure_lane_buffer(ctx, ln->d_trunc, 3 * (mp + 1), "the truncate buffers");
    if (!rc && chunk) rc = ensure_lane_buffer(ctx, ln->d_chunk_offs, lane_offsets_alloc(mp, kMaxPipeChunks) + CFBPE_MAX_DEVICES, "the chunk offsets");
    if (!rc && lens) rc = ensure_lane_buffer(ctx, ln->d_unit_lens, mp + 1, "the unit lengths");
    return rc;
}

// A host unit-start call (cfbpe_encode_batch_char_starts): the starts go where byte starts go (the lane's starts buffer, then
// out_starts), in code points or UTF-16 units; lens (nullable) gets every prompt's length in them.  Under `defer` (a shard of a
// multi-device call) lens is only a flag: the lengths stay in the lane's buffer at the shard's prompt indices.
struct UnitArgs { uint32_t utf16; uint32_t* lens; };
// prompts p0 .. of the call in the lane's length buffer (a sub-batch's prompts keep their index in the call)
UnitView lane_unit_view(Lane* ln, const UnitArgs& u, uint32_t p0) { return UnitView{u.utf16, u.lens ? ln->d_unit_lens.get() + p0 : nullptr}; }
int download_lens(cfbpe_ctx* ctx, Lane* ln, uint32_t* lens, uint32_t p0, uint32_t n, cudaStream_t s) {
    if (lens && n) CK(cudaMemcpyAsync(lens + p0, ln->d_unit_lens.get() + p0, static_cast<uint64_t>(n) * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    return CFBPE_OK;
}

// A host truncate call (cfbpe_truncate_batch): budgets in, cuts and kept counts out, one per prompt of the call.  The ids it needs go to
// the lane's id buffer and are never downloaded.
struct TruncateArgs { const uint32_t* budgets; uint32_t tail; uint32_t* cut; uint32_t* kept; };
TruncateArgs truncate_from(const TruncateArgs& t, uint32_t p0) { return TruncateArgs{t.budgets + p0, t.tail, t.cut + p0, t.kept + p0}; }

// prompts p0 .. of the call in the lane's truncate buffers (a sub-batch's prompts keep their index in the call)
TruncateView lane_truncate_view(cfbpe_ctx* ctx, Lane* ln, uint32_t tail, uint32_t p0) {
    const uint64_t m = static_cast<uint64_t>(ctx->max_prompts) + 1;
    return TruncateView{ln->d_trunc.get() + p0, tail, ln->d_trunc.get() + m + p0, ln->d_trunc.get() + 2 * m + p0};
}
int upload_budgets(cfbpe_ctx* ctx, Lane* ln, const TruncateArgs& t, uint32_t p0, uint32_t n, cudaStream_t s) {
    if (n) CK(cudaMemcpyAsync(ln->d_trunc.get() + p0, t.budgets + p0, static_cast<uint64_t>(n) * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    return CFBPE_OK;
}
int download_cuts(cfbpe_ctx* ctx, Lane* ln, const TruncateArgs& t, uint32_t p0, uint32_t n, cudaStream_t s) {
    if (!n) return CFBPE_OK;
    const TruncateView v = lane_truncate_view(ctx, ln, t.tail, p0);
    CK(cudaMemcpyAsync(t.cut + p0, v.cut, static_cast<uint64_t>(n) * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(t.kept + p0, v.kept, static_cast<uint64_t>(n) * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    return CFBPE_OK;
}

// A host chunk call (cfbpe_chunk_batch): n tokens a chunk, a new chunk every step tokens; spans (room for cap chunks) and chunk
// offsets out.  The ids and starts it needs go to the lane's buffers and are never downloaded.  sub_end (nullable, a shard of a
// multi-device call): gets every sub-batch's chunk_end (shard-local ranks), for the downloads after the shards' totals are known.
struct ChunkArgs { uint32_t n, step; uint32_t* spans; uint64_t cap; uint64_t* offsets; uint64_t* sub_end; };

uint64_t* lane_chunk_totals(cfbpe_ctx* ctx, Lane* ln) { return ln->d_chunk_offs.get() + lane_offsets_alloc(ctx->max_prompts, kMaxPipeChunks); }
// a host call's chunks of the (sub-)batch with workspace w and offsets at q0: the offsets to the lane's buffer, the spans staged
// in w's per-byte scratch, which is dead once the ids are out (begins in ids_by_pos, ends in dense.by_piece: a (sub-)batch has
// no more chunks than tokens and no more tokens than bytes); base: the previous sub-batch's chunk_end, or nullptr
ChunkView lane_chunk_view(Lane* ln, const Workspace& w, uint64_t q0, const uint64_t* base, const ChunkArgs& c) {
    return ChunkView{c.n, c.step, ln->d_chunk_offs.get() + q0, base, w.ids_by_pos, w.dense.by_piece, 1u, UINT64_MAX};
}
// chunks [first, first + count) of the call, staged by lane_chunk_view in w, to their (begin, end) pairs in spans
int download_spans(cfbpe_ctx* ctx, const Workspace& w, uint32_t* spans, uint64_t first, uint64_t count, cudaStream_t s) {
    if (!count) return CFBPE_OK;
    CK(cudaMemcpy2DAsync(spans + 2 * first, 2 * sizeof(uint32_t), w.ids_by_pos, sizeof(uint32_t), sizeof(uint32_t), count, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpy2DAsync(spans + 2 * first + 1, 2 * sizeof(uint32_t), w.dense.by_piece, sizeof(uint32_t), sizeof(uint32_t), count, cudaMemcpyDeviceToHost, s));
    return CFBPE_OK;
}
// the call's `need` chunks exceed chunk_cap; the host learns it in offsets[n]
int fail_chunk_nospace(cfbpe_ctx* ctx, uint64_t need, uint64_t* offsets, uint32_t n) {
    if (offsets) offsets[n] = need;
    return fail(ctx, CFBPE_ENOSPC, "chunk_cap too small: need " + std::to_string(need) + " chunks");
}

// an asynchronous device-path call may still own the lane's workspace: wait for it (the caller has selected the lane's device)
int wait_for_device_call(cfbpe_ctx* ctx, Lane* ln) {
    if (ln->ws_pending) { CK(cudaEventSynchronize(ln->ev_ws.get())); ln->ws_pending = false; }
    return CFBPE_OK;
}

// the inputs of a one-pass host call into the lane's buffers, on s; *b: the batch as the kernels see it
int upload_batch(cfbpe_ctx* ctx, Lane* ln, uint32_t n, const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids, uint64_t total,
                 cudaStream_t s, BatchView* b) {
    if (total) CK(cudaMemcpyAsync(ln->d_bytes.get(), bytes, total, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(ln->d_offsets.get(), offsets, (static_cast<uint64_t>(n) + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
    if (vocab_ids && n) CK(cudaMemcpyAsync(ln->d_vocab_ids.get(), vocab_ids, n, cudaMemcpyHostToDevice, s));
    *b = BatchView{ln->d_bytes.get(), ln->d_offsets.get(), vocab_ids ? ln->d_vocab_ids.get() : nullptr, n, total};
    return CFBPE_OK;
}

// Pipelined host call: the batch is cut into sub-batches of ~kPipeChunkBytes on prompt boundaries; each is an
// independent encode pass on its own slice of the workspace.  Uploads (h2d_stream) run ahead of the kernels
// (stream), downloads (d2h_stream) trail them; token ranks are chained on the device (DeviceStatus::tok_end), so
// ids and offsets land at their final places.  The host only waits for each sub-batch's status to learn how many
// ids to fetch.
// defer != nullptr (a shard of a multi-device call): nothing is downloaded here -- ids, offsets and counts stay in the lane's device
// buffers (dense, shard-local ranks: sub-batch k's offsets at d_out_offsets + sub_batch_offsets_at(p_k, k)) and *defer gets the
// shard's token total.  trunc (nullable): a truncate call; its cuts and kept counts are final (per prompt, prompt-relative) and
// are downloaded under `defer` too.  chunk (nullable): a chunk call; chunk offsets chain across the sub-batches on the device as
// token ranks do (DeviceStatus::chunk_end), so sub-batch k's tile_scan waits for k - 1's whole back stage rather than its scan.
// Under `defer` its offsets and spans stay on the device and chunk->sub_end gets every sub-batch's chunk_end.
int run_host_pipelined(cfbpe_ctx* ctx, DeviceCtx* const* dvs, Lane* const* lns, int G, uint32_t n, const uint8_t* bytes, const uint64_t* offsets,
                       const uint8_t* vocab_ids, uint32_t* out_ids, uint32_t* out_starts, uint64_t out_cap, uint64_t* out_offsets, uint32_t* out_counts,
                       bool want_ids, uint64_t total, uint64_t* defer, uint32_t* cut_out, int* nc_out, const TruncateArgs* trunc,
                       const ChunkArgs* chunk, const UnitArgs* unit = nullptr) {
    // ---- cut
    uint32_t cut[kMaxPipeChunks + 1];
    const int nc = plan_sub_batches(offsets, n, total, ctx->pipe_chunk, kMaxPipeChunks, cut);
    // Sub-batch k runs on device k mod G (G = 1: the single-device call).  Every device keeps the layout of the whole batch
    // (same slices of its own workspace), so the devices differ only in WHICH sub-batches they fill in; the one thing a sub-batch
    // needs from its predecessor -- the token rank it starts at -- is read from the predecessor's device over NVLink (peer
    // memory), behind a cross-device event.  Uploads and downloads of the devices run side by side on their own PCIe links.
    Lane* ln = lns[0];                       // (host-side staging of the offsets and the trace live in the first lane)
    // local offsets of every sub-batch, staged in pinned memory in the device layout
    for (int k = 0; k < nc; ++k) {
        const uint32_t p0 = cut[k], p1 = cut[k + 1];
        const uint64_t o0 = offsets[p0];
        uint64_t* dst = ln->h_offs_stage.get() + sub_batch_offsets_at(p0, k);
        for (uint32_t i = p0; i <= p1; ++i) dst[i - p0] = offsets[i] - o0;
    }
    // ---- enqueue everything that does not depend on the host knowing a result
    const bool trace = G == 1 && getenv("CFBPE_PIPE_TRACE") != nullptr;
    const bool no_copy = trace && getenv("CFBPE_PIPE_NO_COPY") != nullptr;   // measurement aid: the kernels of a pipelined call without its copies (the device buffers still hold the previous call's data)
    if (trace && ln->trace.empty()) {
        ln->trace.resize(kMaxPipeChunks + 1);
        for (auto& events : ln->trace) for (Event& e : events) make_event(e, cudaEventDefault);
    }
    if (trace) CK(cudaEventRecord(ln->trace[nc][0].get(), ln->h2d_stream.get()));
    const auto host_t0 = std::chrono::steady_clock::now();
    auto host_ms = [&]() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - host_t0).count(); };
    double host_enq[kMaxPipeChunks] = {}, host_dl[kMaxPipeChunks] = {};
    for (int k = 0; k < nc; ++k) {
        DeviceCtx* const dv = dvs[k % G];
        Lane* const ln = lns[k % G];
        Lane* const prev = k ? lns[(k - 1) % G] : nullptr;
        if (G > 1) CK(cudaSetDevice(dv->device));
        cudaStream_t cs = ln->stream.get(), hs = ln->h2d_stream.get();
        const uint32_t p0 = cut[k], p1 = cut[k + 1], nk = p1 - p0;
        const uint64_t o0 = offsets[p0], len = offsets[p1] - o0, q0 = sub_batch_offsets_at(p0, k);
        uint8_t* const d_sub = ln->d_bytes.get() + sub_batch_bytes_at(o0, k);
        if (len && !no_copy) CK(cudaMemcpyAsync(d_sub, bytes + o0, len, cudaMemcpyHostToDevice, hs));
        CK(cudaMemcpyAsync(ln->d_offsets.get() + q0, lns[0]->h_offs_stage.get() + q0, (static_cast<uint64_t>(nk) + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, hs));
        if (vocab_ids && nk) CK(cudaMemcpyAsync(ln->d_vocab_ids.get() + p0, vocab_ids + p0, nk, cudaMemcpyHostToDevice, hs));
        if (trunc) { const int rc = upload_budgets(ctx, ln, *trunc, p0, nk, hs); if (rc) return rc; }
        CK(cudaEventRecord(ln->ev_h2d[k].get(), hs));
        if (trace) CK(cudaEventRecord(ln->trace[k][0].get(), hs));
        const int fk = k < kFrontStreams ? k : kFrontStreams - 1;
        cudaStream_t ck = fk ? ln->front[fk].get() : cs;
        const int lv = ln->prio_mode == 2 ? (k * ln->prio_levels) / nc : 0;
        if (ln->prio_mode) ck = ln->pool[lv][(3 * k + 2) % kPoolSlots].get();   // the short-piece kernels of sub-batch k: priority falls with k (earlier sub-batches finish, and download, first)
        Workspace w = slice_workspace(ln->ws, o0, len, static_cast<uint32_t>(k));
        w.status = ln->d_status_arr.get() + k;
        BatchView b{d_sub, ln->d_offsets.get() + q0, vocab_ids ? ln->d_vocab_ids.get() + p0 : nullptr, nk, len};
        // split, long pieces and the back stage run on a top-priority stream of their own: the long-piece kernels are a latency
        // chain that uses little of the machine, so they start as early as possible and the short-piece kernels fill the rest
        cudaStream_t ss = ln->prio_mode ? ln->pool[lv][(3 * k) % kPoolSlots].get() : ln->side[k % kSideStreams].get();
        CK(cudaStreamWaitEvent(ss, ln->ev_h2d[k].get(), 0));
        enqueue_split(b, dv->vs, dv->uc, w, ss, static_cast<ProfEvents*>(nullptr), static_cast<uint32_t>(dv->sm_count));
        CK(cudaEventRecord(ln->ev_scan[k].get(), ss));
        if (trace) CK(cudaEventRecord(ln->trace[k][1].get(), ss));
        CK(cudaStreamWaitEvent(ck, ln->ev_scan[k].get(), 0));
        cudaStream_t ss2 = ln->prio_mode ? ln->pool[lv][(3 * k + 1) % kPoolSlots].get() : ln->side2[k % kSideStreams].get();
        CK(cudaStreamWaitEvent(ss2, ln->ev_scan[k].get(), 0));
        enqueue_list(b, dv->vs, w, static_cast<uint32_t>(dv->sm_count * 4), ss2, static_cast<ProfEvents*>(nullptr));   // the big pieces, beside everything else
        CK(cudaEventRecord(ln->ev_list[k].get(), ss2));
        if (trace) CK(cudaEventRecord(ln->trace[k][6].get(), ss2));
        enqueue_long(b, dv->vs, w, static_cast<uint32_t>(dv->sm_count * 4), ss, static_cast<ProfEvents*>(nullptr));   // tail overlaps what follows on cs
        if (trace) CK(cudaEventRecord(ln->trace[k][3].get(), ss));
        enqueue_short(b, dv->vs, w, static_cast<uint32_t>(dv->sm_count * 4), ck, static_cast<ProfEvents*>(nullptr));
        CK(cudaEventRecord(ln->ev_front[k].get(), ck));
        if (trace) CK(cudaEventRecord(ln->trace[k][2].get(), ck));
        CK(cudaStreamWaitEvent(ss, ln->ev_front[k].get(), 0));
        CK(cudaStreamWaitEvent(ss, ln->ev_list[k].get(), 0));
        enqueue_count(b, w, ss, static_cast<ProfEvents*>(nullptr));
        if (trace) CK(cudaEventRecord(ln->trace[k][7].get(), ss));
        if (k) CK(cudaStreamWaitEvent(ss, prev->ev_chain[k - 1].get(), 0));    // token ranks chain through DeviceStatus::tok_end: only the scan waits
        enqueue_scan(b, w, ss, static_cast<ProfEvents*>(nullptr), k ? &prev->d_status_arr.get()[k - 1].tok_end : nullptr);   // (G > 1: a peer pointer)
        if (!chunk) CK(cudaEventRecord(ln->ev_chain[k].get(), ss));
        const TruncateView tv = trunc ? lane_truncate_view(ctx, ln, trunc->tail, p0) : TruncateView{};
        const ChunkView cv = chunk ? lane_chunk_view(ln, w, q0, k ? &prev->d_status_arr.get()[k - 1].chunk_end : nullptr, *chunk) : ChunkView{};
        const UnitView uv = unit ? lane_unit_view(ln, *unit, p0) : UnitView{};
        enqueue_emit(b, w, want_ids ? ln->d_out_ids.get() : nullptr, ctx->max_bytes, ln->d_out_offsets.get() + q0, ln->d_out_counts.get() + p0,
                     ss, static_cast<ProfEvents*>(nullptr), (out_starts || chunk) ? ln->d_out_starts.get() : nullptr, &dv->vs, trunc ? &tv : nullptr,
                     chunk ? &cv : nullptr, unit ? &uv : nullptr);
        if (chunk) CK(cudaEventRecord(ln->ev_chain[k].get(), ss));       // (the chunk scan read the previous chunk_end: the chain ends here)
        CK(cudaGetLastError());
        status_publish_kernel<<<1, 64, 0, ss>>>(ln->d_status_arr.get() + k, ln->h_status_arr.get() + k);
        CK(cudaEventRecord(ln->ev_done[k].get(), ss));
        if (trace) { CK(cudaEventRecord(ln->trace[k][4].get(), ss)); host_enq[k] = host_ms(); }
    }
    // ---- trail the kernels with the downloads
    int err = CFBPE_OK;
    uint64_t tok_total = 0, chunk_total = 0;
    for (int k = 0; k < nc; ++k) {
        Lane* const ln = lns[k % G];
        if (G > 1) CK(cudaSetDevice(dvs[k % G]->device));
        cudaStream_t ds = ln->d2h_stream.get();
        CK(cudaEventSynchronize(ln->ev_done[k].get()));
        const DeviceStatus st = ln->h_status_arr.get()[k];
        const uint32_t p0 = cut[k], p1 = cut[k + 1], nk = p1 - p0;
        if (!err) err = fail_status(ctx, st);
        const uint64_t base = st.tok_end - st.n_tokens;
        tok_total = st.tok_end;
        if (!err && trunc) { const int rc = download_cuts(ctx, ln, *trunc, p0, nk, ds); if (rc) return rc; }
        if (chunk) { chunk_total = st.chunk_end; if (chunk->sub_end) chunk->sub_end[k] = st.chunk_end; }
        if (err || defer) continue;
        if (no_copy) continue;
        if (chunk) {
            const uint64_t q0 = sub_batch_offsets_at(p0, k);
            CK(cudaMemcpyAsync(chunk->offsets + p0, ln->d_chunk_offs.get() + q0, (static_cast<uint64_t>(nk) + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, ds));
            if (st.chunk_end <= chunk->cap) {
                const Workspace w = slice_workspace(ln->ws, offsets[p0], offsets[p1] - offsets[p0], static_cast<uint32_t>(k));
                if (const int rc = download_spans(ctx, w, chunk->spans, st.chunk_end - st.n_chunks, st.n_chunks, ds)) return rc;
            }
        }
        if (want_ids && out_ids && st.tok_end <= out_cap && st.n_tokens)
            CK(cudaMemcpyAsync(out_ids + base, ln->d_out_ids.get() + base, st.n_tokens * sizeof(uint32_t), cudaMemcpyDeviceToHost, ds));
        if (out_starts && st.tok_end <= out_cap && st.n_tokens)      // (prompt-relative: the same ranks and base as the ids)
            CK(cudaMemcpyAsync(out_starts + base, ln->d_out_starts.get() + base, st.n_tokens * sizeof(uint32_t), cudaMemcpyDeviceToHost, ds));
        if (out_offsets) CK(cudaMemcpyAsync(out_offsets + p0, ln->d_out_offsets.get() + sub_batch_offsets_at(p0, k), (static_cast<uint64_t>(nk) + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, ds));
        if (out_counts && nk) CK(cudaMemcpyAsync(out_counts + p0, ln->d_out_counts.get() + p0, static_cast<uint64_t>(nk) * sizeof(uint32_t), cudaMemcpyDeviceToHost, ds));
        if (unit) { const int rc = download_lens(ctx, ln, unit->lens, p0, nk, ds); if (rc) return rc; }
        if (trace) { CK(cudaEventRecord(ln->trace[k][5].get(), ds)); host_dl[k] = host_ms(); }
    }
    for (int g = 0; g < G; ++g) {
        Lane* const lg = lns[g];
        if (G > 1) CK(cudaSetDevice(dvs[g]->device));
        CK(cudaStreamSynchronize(lg->d2h_stream.get()));
        CK(cudaStreamSynchronize(lg->stream.get()));
        for (int k = 1; k < kFrontStreams; ++k) CK(cudaStreamSynchronize(lg->front[k].get()));
        for (int k = 0; k < kSideStreams; ++k) CK(cudaStreamSynchronize(lg->side[k].get()));
        for (int k = 0; k < kSideStreams; ++k) CK(cudaStreamSynchronize(lg->side2[k].get()));
        if (lg->prio_mode) for (int l = 0; l < kPrioLevels; ++l) for (int j = 0; j < kPoolSlots; ++j) if (lg->pool[l][j]) CK(cudaStreamSynchronize(lg->pool[l][j].get()));
    }
    if (trace && !err) {
        fprintf(stderr, "pipe trace (ms since the first upload was enqueued): sub-batch bytes | h2d split long_end list_end short count back d2h\n");
        for (int k = 0; k < nc; ++k) {
            float t[kTracePoints] = {};
            for (int j = 0; j < kTracePoints; ++j) if (!(no_copy && j == 5)) cudaEventElapsedTime(&t[j], ln->trace[nc][0].get(), ln->trace[k][j].get());
            fprintf(stderr, "  %2d %9llu | %6.2f %6.2f %6.2f %6.2f %6.2f %6.2f %6.2f %6.2f | host: enqueued %.2f download issued %.2f\n", k,
                    static_cast<unsigned long long>(offsets[cut[k + 1]] - offsets[cut[k]]), t[0], t[1], t[3], t[6], t[2], t[7], t[4], t[5], host_enq[k], host_dl[k]);
        }
    }
    if (err) return err;
    if (defer) { *defer = tok_total; if (cut_out) { std::memcpy(cut_out, cut, sizeof(uint32_t) * (nc + 1)); *nc_out = nc; } return CFBPE_OK; }
    if (want_ids && tok_total > out_cap) return fail_nospace(ctx, tok_total, out_offsets, n);
    if (chunk && chunk_total > chunk->cap) return fail_chunk_nospace(ctx, chunk_total, chunk->offsets, n);
    return CFBPE_OK;
}

// One device's share of a host call (the whole call on a single-device context): validation is done, the lane is locked.
// defer / cut_out / nc_out: see run_host_pipelined; the one-shot path under `defer` leaves everything on the device as ONE sub-batch.
// out_starts != nullptr: the tokens' starts too (in ln->d_out_starts, beside the ids; under `defer` it is only a flag).
// trunc != nullptr: a truncate call (the ids stay in the lane; the cuts and kept counts are downloaded, under `defer` too).
// chunk != nullptr: a chunk call (the ids and starts stay in the lane; the chunk offsets and spans are downloaded, except under
// `defer`, where chunk->sub_end[0] gets the chunk total).
// unit != nullptr: a unit-start call (out_starts gets the unit starts; the lengths are downloaded, except under `defer`).
int run_lane(cfbpe_ctx* ctx, DeviceCtx* dv, Lane* ln, uint32_t n, const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids,
             uint32_t* out_ids, uint32_t* out_starts, uint64_t out_cap, uint64_t* out_offsets, uint32_t* out_counts, bool want_ids, uint64_t total,
             uint64_t* defer = nullptr, uint32_t* cut_out = nullptr, int* nc_out = nullptr, const TruncateArgs* trunc = nullptr,
             const ChunkArgs* chunk = nullptr, const UnitArgs* unit = nullptr) {
    CK(cudaSetDevice(dv->device));
    int rc = wait_for_device_call(ctx, ln);
    if (!rc) rc = ensure_call_buffers(ctx, ln, out_starts || chunk, trunc != nullptr, chunk != nullptr, unit && unit->lens);
    if (rc) return rc;
    const bool profiling = ctx->profiling.load();
    if (!profiling && total >= ctx->pipe_min && n >= 2)
        return run_host_pipelined(ctx, &dv, &ln, 1, n, bytes, offsets, vocab_ids, out_ids, out_starts, out_cap, out_offsets, out_counts, want_ids, total,
                                  defer, cut_out, nc_out, trunc, chunk, unit);
    cudaStream_t s = ln->stream.get();
    ProfEvents* prof = profiling ? &ln->prof : nullptr;
    if (prof) { std::memset(prof->launched, 0, sizeof prof->launched); cudaEventRecord(prof->total[0].get(), s); cudaEventRecord(prof->h2d[0].get(), s); }
    BatchView b;
    rc = upload_batch(ctx, ln, n, bytes, offsets, vocab_ids, total, s, &b);
    if (!rc && trunc) rc = upload_budgets(ctx, ln, *trunc, 0, n, s);
    if (rc) return rc;
    if (prof) cudaEventRecord(prof->h2d[1].get(), s);

    const TruncateView tv = trunc ? lane_truncate_view(ctx, ln, trunc->tail, 0) : TruncateView{};
    const ChunkView cv = chunk ? lane_chunk_view(ln, ln->ws, 0, nullptr, *chunk) : ChunkView{};
    const UnitView uv = unit ? lane_unit_view(ln, *unit, 0) : UnitView{};
    enqueue_encode(b, dv->vs, dv->uc, ln->ws, want_ids ? ln->d_out_ids.get() : nullptr, ctx->max_bytes, ln->d_out_offsets.get(),
                   ln->d_out_counts.get(), static_cast<uint32_t>(dv->sm_count * 4), s, prof ? s : ln->aux_stream.get(), prof ? s : ln->aux2_stream.get(),
                   ln->ev_fork.get(), ln->ev_join.get(), ln->ev_join2.get(), prof, nullptr, (out_starts || chunk) ? ln->d_out_starts.get() : nullptr, trunc ? &tv : nullptr,
                   chunk ? &cv : nullptr, unit ? &uv : nullptr);
    CK(cudaGetLastError());
    if (prof) cudaEventRecord(prof->d2h[0].get(), s);
    CK(cudaMemcpyAsync(ln->h_status.get(), ln->ws.status, sizeof(DeviceStatus), cudaMemcpyDeviceToHost, s));
    if (trunc && (rc = download_cuts(ctx, ln, *trunc, 0, n, s))) return rc;
    if (!defer) {
        if (out_offsets) CK(cudaMemcpyAsync(out_offsets, ln->d_out_offsets.get(), (static_cast<uint64_t>(n) + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
        if (out_counts && n) CK(cudaMemcpyAsync(out_counts, ln->d_out_counts.get(), static_cast<uint64_t>(n) * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        if (chunk) CK(cudaMemcpyAsync(chunk->offsets, ln->d_chunk_offs.get(), (static_cast<uint64_t>(n) + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
        if (unit && (rc = download_lens(ctx, ln, unit->lens, 0, n, s))) return rc;
    }
    CK(cudaStreamSynchronize(s));
    const DeviceStatus st = *ln->h_status;
    if ((rc = fail_status(ctx, st))) return rc;
    if (defer) {
        *defer = st.n_tokens;
        if (cut_out) { cut_out[0] = 0; cut_out[1] = n; *nc_out = 1; }
        if (chunk && chunk->sub_end) chunk->sub_end[0] = st.chunk_end;
        return CFBPE_OK;
    }
    if (chunk) {
        if (st.chunk_end > chunk->cap) return fail_chunk_nospace(ctx, st.chunk_end, chunk->offsets, n);
        if ((rc = download_spans(ctx, ln->ws, chunk->spans, 0, st.chunk_end, s))) return rc;
    }
    if (want_ids) {
        if (st.n_tokens > out_cap) return fail_nospace(ctx, st.n_tokens, out_offsets, n);
        if (out_ids && st.n_tokens) CK(cudaMemcpyAsync(out_ids, ln->d_out_ids.get(), st.n_tokens * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        if (out_starts && st.n_tokens) CK(cudaMemcpyAsync(out_starts, ln->d_out_starts.get(), st.n_tokens * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    }
    if (prof) { cudaEventRecord(prof->d2h[1].get(), s); cudaEventRecord(prof->total[1].get(), s); }
    CK(cudaStreamSynchronize(s));
    if (prof) fill_profile(ln, total);
    return CFBPE_OK;
}

// ---------------------------------------------------------------------------------------
// special tokens (specials.h, specials.cuh)
// ---------------------------------------------------------------------------------------
int fail_disallowed(cfbpe_ctx* ctx, uint32_t prompt, uint32_t vid, uint32_t k, uint32_t* out_bad) {
    if (out_bad) { out_bad[0] = prompt; out_bad[1] = k; }
    std::string tok;
    const std::vector<uint32_t>& w = ctx->specials[vid < CFBPE_MAX_VOCABS ? vid : 0];
    if (!w.empty() && k < w[0]) {
        const uint8_t* sb = reinterpret_cast<const uint8_t*>(w.data() + w[11]);
        tok.assign(reinterpret_cast<const char*>(sb + w[w[8] + k]), w[w[8] + k + 1] - w[w[8] + k]);
    }
    return fail(ctx, CFBPE_EBADMSG, "prompt " + std::to_string(prompt) + " holds the special token " + tok + " (index " + std::to_string(k) +
                                    "), which this call disallows");
}

// the lane's special buffers, all or none: they are built aside and installed once every allocation succeeded (on a failure, what
// was allocated is released on return).  The caller has selected the lane's device.
int ensure_special_lane(cfbpe_ctx* ctx, Lane* ln) {
    if (ln->sp.h_status) return CFBPE_OK;
    const uint64_t mp = ctx->max_prompts;
    LaneSpecial sp;
    bool ok = dmalloc(sp.kept_n, mp + 1) == cudaSuccess;
    ok = ok && dmalloc(sp.kept_base, mp + 1) == cudaSuccess;
    ok = ok && dmalloc(sp.st_off, mp + 2) == cudaSuccess;
    ok = ok && dmalloc(sp.st_vocab, mp + 1) == cudaSuccess;
    ok = ok && dmalloc(sp.st_id, mp + 1) == cudaSuccess;
    ok = ok && dmalloc(sp.st_base, mp + 1) == cudaSuccess;
    ok = ok && dmalloc(sp.fin_offsets, mp + 1) == cudaSuccess;
    ok = ok && dmalloc(sp.fin_counts, mp + 1) == cudaSuccess;
    ok = ok && dmalloc(sp.modes, static_cast<uint64_t>(CFBPE_MAX_VOCABS) * kMaxSpecials) == cudaSuccess;
    ok = ok && dmalloc(sp.status, 1) == cudaSuccess;
    ok = ok && hmalloc(sp.h_status, 1) == cudaSuccess;
    if (!ok) { cudaGetLastError(); return fail(ctx, CFBPE_ENOMEM, "no device memory for the special-token buffers"); }
    ln->sp = std::move(sp);
    return CFBPE_OK;
}

SpecialWork special_work(Lane* ln) {
    const LaneSpecial& sp = ln->sp;
    return SpecialWork{sp.kept_n.get(), sp.kept_base.get(), sp.st_off.get(), sp.st_vocab.get(), sp.st_id.get(), sp.st_base.get(), sp.status.get()};
}

// The special set of one call on device dv (fill_special_set), with the lane's special buffers allocated and the call's mode bytes
// uploaded into them.  *scan = false: no vocabulary looks for any special, the call is the ordinary path.
int special_set(cfbpe_ctx* ctx, DeviceCtx* dv, Lane* ln, const uint8_t* const* modes, SpecialSet* out, bool* scan, cudaStream_t s) {
    int rc = ensure_special_lane(ctx, ln);
    if (rc) return rc;
    const uint32_t* words[CFBPE_MAX_VOCABS];
    for (uint32_t v = 0; v < CFBPE_MAX_VOCABS; ++v) words[v] = ctx->specials[v].empty() ? nullptr : ctx->specials[v].data();
    uint32_t bad[2];
    if (fill_special_set(words, dv->specials.v, modes, out, scan, bad))
        return fail(ctx, CFBPE_EINVAL, "modes[" + std::to_string(bad[0]) + "][" + std::to_string(bad[1]) + "] is not a CFBPE_SPECIAL_* value");
    for (uint32_t v = 0; v < CFBPE_MAX_VOCABS; ++v) {
        if (!out->modes[v]) continue;
        uint8_t* dm = ln->sp.modes.get() + static_cast<uint64_t>(v) * kMaxSpecials;
        CK(cudaMemcpyAsync(dm, out->modes[v], words[v][0], cudaMemcpyHostToDevice, s));
        out->modes[v] = dm;
    }
    return CFBPE_OK;
}

// Where the ids, offsets and counts of an encode pass go
struct EncodeOut { uint32_t* ids; uint64_t cap; uint64_t* offsets; uint32_t* counts; };

// The rest of a special call once its batch is on the device and special_set has run: the scan (when some vocabulary looks for a
// special) and what it found, then the ordinary path on the prompts as they are, into `plain`, or on the stretches followed by the
// splice, into `spliced` (the stretches' own ids, offsets and counts go to the lane's d_out_* buffers).  *did_splice: which ran.
int enqueue_special_call(cfbpe_ctx* ctx, DeviceCtx* dv, Lane* ln, const BatchView& b, const SpecialSet& sp, bool scan, cudaStream_t s,
                         const EncodeOut& plain, const EncodeOut& spliced, uint32_t* out_bad, bool* did_splice) {
    const SpecialWork sw = special_work(ln);
    uint64_t n_str = b.n_prompts;
    if (scan) {       // the one synchronisation of the call: the host needs the number of stretches for the launch geometry
        enqueue_special_scan(b, sp, ln->ws, sw, s);
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(ln->sp.h_status.get(), ln->sp.status.get(), sizeof(SpecialStatus), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
        const SpecialScanResult r = special_scan_result(*ln->sp.h_status, b.n_prompts, ctx->max_prompts);
        if (r.disallowed) return fail_disallowed(ctx, r.prompt, r.vocab, r.index, out_bad);
        if (!r.fits)
            return fail(ctx, CFBPE_EINVAL, "n_prompts + 2 x special-token matches (" + std::to_string(r.n_stretches) + ") exceeds max_prompts of this context");
        n_str = r.n_stretches;
    }
    *did_splice = n_str != b.n_prompts;
    const uint32_t grid = static_cast<uint32_t>(dv->sm_count * 4);
    if (!*did_splice) {
        enqueue_encode(b, dv->vs, dv->uc, ln->ws, plain.ids, plain.cap, plain.offsets, plain.counts, grid,
                       s, ln->aux_stream.get(), ln->aux2_stream.get(), ln->ev_fork.get(), ln->ev_join.get(), ln->ev_join2.get(), static_cast<ProfEvents*>(nullptr));
    } else {
        enqueue_encode_special(b, sp, dv->vs, dv->uc, ln->ws, sw, static_cast<uint32_t>(n_str), ln->d_out_ids.get(), ctx->max_bytes, ln->d_out_offsets.get(),
                               ln->d_out_counts.get(), spliced.ids, spliced.cap, spliced.offsets, spliced.counts,
                               grid, s, ln->aux_stream.get(), ln->aux2_stream.get(), ln->ev_fork.get(), ln->ev_join.get(), ln->ev_join2.get(), static_cast<ProfEvents*>(nullptr));
    }
    CK(cudaGetLastError());
    return CFBPE_OK;
}

// offsets of a shard are ranks inside the shard: add the tokens of the shards before it (the all-gathered totals)
__global__ void rebase_offsets_kernel(uint64_t* __restrict__ offsets, uint64_t n, const uint64_t* __restrict__ totals, uint32_t shard) {
    uint64_t base = 0;
    for (uint32_t d = 0; d < shard; ++d) base += totals[d];
    const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) offsets[i] += base;
}

// A host call on a multi-device context: the batch is cut into one contiguous range of whole prompts per device, balanced by
// bytes; every device runs its shard on its own host thread and lane (uploads, kernels), the per-shard token totals are
// all-gathered with NCCL (8 bytes a device: the path's only exchange), every device rebases its offsets by the totals of the
// shards before it and downloads ids, offsets and counts straight to their final places in the caller's buffers.
int run_lane_special(cfbpe_ctx* ctx, DeviceCtx* dv, Lane* ln, uint32_t n, const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids,
                     const uint8_t* const* modes, uint32_t* out_ids, uint64_t out_cap, uint64_t* out_offsets, uint32_t* out_counts, bool want_ids,
                     uint64_t total, uint32_t* out_bad, uint64_t* defer);
int run_lane_lossy(cfbpe_ctx* ctx, DeviceCtx* dv, Lane* ln, uint32_t n, const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids,
                   uint32_t* out_ids, uint64_t out_cap, uint64_t* out_offsets, uint32_t* out_counts, bool want_ids, uint64_t total,
                   uint32_t* out_replaced, uint64_t* defer);

// special != nullptr: a special-token call (cfbpe_encode_batch_special): every shard runs its own special pass; special->modes
// are the call's modes, special->bad gets the prompt and special index of a CFBPE_EBADMSG
struct SpecialArgs { const uint8_t* const* modes; uint32_t* bad; };
// lossy != nullptr: a lossy call (cfbpe_encode_batch_lossy): every shard runs its own scan and, when it needs one, its own repair;
// lossy->replaced (nullable) gets every prompt's U+FFFD count
struct LossyArgs { uint32_t* replaced; };
int run_multi_device(cfbpe_ctx* ctx, uint32_t n, const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids,
                     uint32_t* out_ids, uint32_t* out_starts, uint64_t out_cap, uint64_t* out_offsets, uint32_t* out_counts, bool want_ids, uint64_t total,
                     const SpecialArgs* special = nullptr, const TruncateArgs* trunc = nullptr, const ChunkArgs* chunk = nullptr,
                     const UnitArgs* unit = nullptr, const LossyArgs* lossy = nullptr) {
    const uint32_t G = static_cast<uint32_t>(ctx->devs.size());
    std::vector<uint32_t> lo(G + 1, 0);
    for (uint32_t d = 1; d < G; ++d) {      // first prompt whose start is >= d * total / G
        const uint64_t target = total / G * d;
        uint32_t a = lo[d - 1], b = n;
        while (a < b) { const uint32_t m = a + (b - a) / 2; if (offsets[m] >= target) b = m; else a = m + 1; }
        lo[d] = a;
    }
    lo[G] = n;
    for (uint32_t d = 0; d < G; ++d)
        if (offsets[lo[d + 1]] - offsets[lo[d]] > ctx->max_bytes) return fail(ctx, CFBPE_EINVAL, "a device's shard exceeds max_batch_bytes (one prompt is too large to balance)");
    struct Shard { int rc = CFBPE_OK; std::string err; uint64_t tokens = 0; std::vector<uint64_t> local_offs; uint32_t cut[kMaxPipeChunks + 1]; int nc = 0; uint32_t bad[2] = {};
                   uint64_t chunk_end[kMaxPipeChunks] = {}; };
    std::vector<Shard> sh(G);
    std::vector<std::unique_ptr<LaneLock>> locks(G);
    for (uint32_t d = 0; d < G; ++d) locks[d].reset(new LaneLock(ctx->devs[d].get()));
    // ---- phase 1: every device encodes its shard; results stay on the device
    {
        std::vector<std::thread> th;
        for (uint32_t d = 0; d < G; ++d) th.emplace_back([&, d]() {
            Shard& s = sh[d];
            const uint32_t p0 = lo[d], nd = lo[d + 1] - lo[d];
            const uint64_t o0 = offsets[p0];
            s.local_offs.resize(static_cast<size_t>(nd) + 1);
            for (uint32_t i = 0; i <= nd; ++i) s.local_offs[i] = offsets[p0 + i] - o0;
            if (special) {
                s.rc = run_lane_special(ctx, ctx->devs[d].get(), locks[d]->ln, nd, bytes + o0, s.local_offs.data(), vocab_ids ? vocab_ids + p0 : nullptr,
                                        special->modes, nullptr, 0, nullptr, nullptr, want_ids, s.local_offs[nd], s.bad, &s.tokens);
                s.cut[0] = 0; s.cut[1] = nd; s.nc = 1;
            } else if (lossy) {
                s.rc = run_lane_lossy(ctx, ctx->devs[d].get(), locks[d]->ln, nd, bytes + o0, s.local_offs.data(), vocab_ids ? vocab_ids + p0 : nullptr,
                                      nullptr, 0, nullptr, nullptr, want_ids, s.local_offs[nd], nullptr, &s.tokens);
                s.cut[0] = 0; s.cut[1] = nd; s.nc = 1;
            } else {
                const TruncateArgs shard_trunc = trunc ? truncate_from(*trunc, p0) : TruncateArgs{};
                const ChunkArgs shard_chunk = chunk ? ChunkArgs{chunk->n, chunk->step, nullptr, UINT64_MAX, nullptr, s.chunk_end} : ChunkArgs{};
                s.rc = run_lane(ctx, ctx->devs[d].get(), locks[d]->ln, nd, bytes + o0, s.local_offs.data(), vocab_ids ? vocab_ids + p0 : nullptr,
                                nullptr, out_starts, 0, nullptr, nullptr, want_ids, s.local_offs[nd], &s.tokens, s.cut, &s.nc,
                                trunc ? &shard_trunc : nullptr, chunk ? &shard_chunk : nullptr, unit);
            }
            if (s.rc) s.err = tl_err;
        });
        for (auto& t : th) t.join();
    }
    for (uint32_t d = 0; d < G && special; ++d)        // a disallowed special wins over every other error, the lowest prompt first
        if (sh[d].rc == CFBPE_EBADMSG) {
            const uint32_t p = sh[d].bad[0] + lo[d];
            return fail_disallowed(ctx, p, vocab_ids ? vocab_ids[p] : 0u, sh[d].bad[1], special->bad);
        }
    for (uint32_t d = 0; d < G; ++d) if (sh[d].rc) return fail(ctx, sh[d].rc, sh[d].err);
    // ---- phase 2: all-gather of the token totals (NCCL, 8 bytes a device), rebase, download to the final places
    const NcclApi& nc = ctx->nccl;
    int nrc = nc.GroupStart();
    for (uint32_t d = 0; d < G && nrc == 0; ++d) {
        Lane* ln = locks[d]->ln;
        cudaSetDevice(ctx->devs[d]->device);
        ln->h_totals.get()[CFBPE_MAX_DEVICES] = sh[d].tokens;                                   // (slot past the gathered ones: this shard's own total)
        cudaMemcpyAsync(ln->d_totals.get() + CFBPE_MAX_DEVICES, ln->h_totals.get() + CFBPE_MAX_DEVICES, sizeof(uint64_t), cudaMemcpyHostToDevice, ln->stream.get());
        nrc = nc.AllGather(ln->d_totals.get() + CFBPE_MAX_DEVICES, ln->d_totals.get(), 1, kNcclUint64, ctx->devs[d]->comm, ln->stream.get());
    }
    { const int r2 = nc.GroupEnd(); if (nrc == 0) nrc = r2; }
    if (nrc != 0) return fail(ctx, CFBPE_EIO, std::string("ncclAllGather of the shard totals: ") + nc.GetErrorString(nrc));
    std::vector<int> rcs(G, CFBPE_OK);
    std::vector<std::string> errs(G);
    uint64_t grand = 0;
    for (uint32_t d = 0; d < G; ++d) grand += sh[d].tokens;
    const bool fits = !want_ids || grand <= out_cap;
    // a chunk call: every shard's chunk total is on the host already (its last sub-batch's chunk_end, shard-local)
    std::vector<uint64_t> chunk_tot(G, 0), chunk_base(G + 1, 0);
    for (uint32_t d = 0; d < G && chunk; ++d) { chunk_tot[d] = sh[d].nc ? sh[d].chunk_end[sh[d].nc - 1] : 0; chunk_base[d + 1] = chunk_base[d] + chunk_tot[d]; }
    const bool chunks_fit = !chunk || chunk_base[G] <= chunk->cap;
    {
        std::vector<std::thread> th;
        for (uint32_t d = 0; d < G; ++d) th.emplace_back([&, d]() {
            Lane* ln = locks[d]->ln;
            const Shard& s = sh[d];
            const uint32_t p0 = lo[d];
            auto ck = [&](cudaError_t e, const char* what) { if (e != cudaSuccess && rcs[d] == CFBPE_OK) { rcs[d] = CFBPE_EIO; errs[d] = std::string(what) + ": " + cudaGetErrorString(e); } };
            ck(cudaSetDevice(ctx->devs[d]->device), "cudaSetDevice");
            cudaStream_t st = ln->stream.get();
            ck(cudaMemcpyAsync(ln->h_totals.get(), ln->d_totals.get(), sizeof(uint64_t) * G, cudaMemcpyDeviceToHost, st), "totals download");
            if (chunk) ck(cudaMemcpyAsync(lane_chunk_totals(ctx, ln), chunk_tot.data(), sizeof(uint64_t) * G, cudaMemcpyHostToDevice, st), "chunk totals upload");
            for (int k = 0; k < s.nc; ++k) {
                const uint32_t q0 = s.cut[k], nk = s.cut[k + 1] - s.cut[k];
                const bool last = (k + 1 == s.nc) && (d + 1 == G);
                const uint64_t cnt = static_cast<uint64_t>(nk) + (last ? 1 : 0);      // the boundary entry belongs to the next sub-batch / shard
                if (!cnt) continue;
                uint64_t* src = ln->d_out_offsets.get() + sub_batch_offsets_at(q0, k);
                rebase_offsets_kernel<<<static_cast<unsigned>((cnt + 255) / 256), 256, 0, st>>>(src, cnt, ln->d_totals.get(), d);
                if (out_offsets) ck(cudaMemcpyAsync(out_offsets + p0 + q0, src, cnt * sizeof(uint64_t), cudaMemcpyDeviceToHost, st), "offsets download");
                if (out_counts && nk) ck(cudaMemcpyAsync(out_counts + p0 + q0, ln->d_out_counts.get() + q0, static_cast<uint64_t>(nk) * sizeof(uint32_t), cudaMemcpyDeviceToHost, st), "counts download");
                if (lossy && lossy->replaced && nk) ck(cudaMemcpyAsync(lossy->replaced + p0 + q0, ln->lossy.replaced.get() + q0, static_cast<uint64_t>(nk) * sizeof(uint32_t), cudaMemcpyDeviceToHost, st), "replaced download");
                if (unit && unit->lens && nk) ck(cudaMemcpyAsync(unit->lens + p0 + q0, ln->d_unit_lens.get() + q0, static_cast<uint64_t>(nk) * sizeof(uint32_t), cudaMemcpyDeviceToHost, st), "lengths download");
                if (chunk) {      // chunk offsets: rebased as the token offsets, by the chunk totals of the shards before; spans: prompt-relative
                    uint64_t* csrc = ln->d_chunk_offs.get() + sub_batch_offsets_at(q0, k);
                    rebase_offsets_kernel<<<static_cast<unsigned>((cnt + 255) / 256), 256, 0, st>>>(csrc, cnt, lane_chunk_totals(ctx, ln), d);
                    ck(cudaMemcpyAsync(chunk->offsets + p0 + q0, csrc, cnt * sizeof(uint64_t), cudaMemcpyDeviceToHost, st), "chunk offsets download");
                    const uint64_t c0 = k ? s.chunk_end[k - 1] : 0, c1 = s.chunk_end[k];
                    if (chunks_fit && c1 > c0) {
                        const uint64_t o0 = s.local_offs[q0];
                        const Workspace w = slice_workspace(ln->ws, o0, s.local_offs[q0 + nk] - o0, static_cast<uint32_t>(k));
                        ck(cudaMemcpy2DAsync(chunk->spans + 2 * (chunk_base[d] + c0), 2 * sizeof(uint32_t), w.ids_by_pos, sizeof(uint32_t), sizeof(uint32_t),
                                             c1 - c0, cudaMemcpyDeviceToHost, st), "span begins download");
                        ck(cudaMemcpy2DAsync(chunk->spans + 2 * (chunk_base[d] + c0) + 1, 2 * sizeof(uint32_t), w.dense.by_piece, sizeof(uint32_t), sizeof(uint32_t),
                                             c1 - c0, cudaMemcpyDeviceToHost, st), "span ends download");
                    }
                }
            }
            ck(cudaStreamSynchronize(st), "stream sync");
            uint64_t base = 0;
            for (uint32_t e = 0; e < d; ++e) base += ln->h_totals.get()[e];
            if (want_ids && out_ids && fits && s.tokens) ck(cudaMemcpyAsync(out_ids + base, ln->d_out_ids.get(), s.tokens * sizeof(uint32_t), cudaMemcpyDeviceToHost, st), "ids download");
            if (out_starts && fits && s.tokens) ck(cudaMemcpyAsync(out_starts + base, ln->d_out_starts.get(), s.tokens * sizeof(uint32_t), cudaMemcpyDeviceToHost, st), "starts download");
            ck(cudaStreamSynchronize(st), "stream sync");
        });
        for (auto& t : th) t.join();
    }
    for (uint32_t d = 0; d < G; ++d) if (rcs[d]) return fail(ctx, rcs[d], errs[d]);
    if (!fits) return fail_nospace(ctx, grand, out_offsets, n);
    if (!chunks_fit) return fail_chunk_nospace(ctx, chunk_base[G], chunk->offsets, n);
    return CFBPE_OK;
}

// shared body of encode_batch / encode_batch_starts / encode_batch_char_starts / count_batch / truncate_batch / chunk_batch (host
// buffers); out_starts: NULL but for encode_batch_starts and encode_batch_char_starts; trunc: NULL but for truncate_batch, chunk: NULL
// but for chunk_batch (both emit the ids into the lane, out_ids NULL, out_cap unlimited); unit: NULL but for encode_batch_char_starts
int run_host(cfbpe_ctx* ctx, uint32_t n, const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids,
             uint32_t* out_ids, uint32_t* out_starts, uint64_t out_cap, uint64_t* out_offsets, uint32_t* out_counts, bool want_ids,
             const TruncateArgs* trunc = nullptr, const ChunkArgs* chunk = nullptr, const UnitArgs* unit = nullptr) {
    tl_err.clear();
    std::shared_lock<std::shared_mutex> vocabs(ctx->vocab_mu);
    uint64_t total = 0;
    int rc = validate_batch(ctx, n, offsets, vocab_ids, &total);
    if (rc) return rc;
    if (total && !bytes) return fail(ctx, CFBPE_EINVAL, "bytes is NULL");
    if (want_ids && !trunc && !chunk && (!out_offsets || (!out_ids && out_cap))) return fail(ctx, CFBPE_EINVAL, "output pointer is NULL");
    if (ctx->devs.size() > 1 && n >= ctx->devs.size() && !ctx->profiling.load()) {
        // Two ways over several devices.  When every device can hold the whole batch (and the devices see each other's memory):
        // the sub-batches of ONE pipelined call go round-robin over the devices -- uploads, kernels and downloads of all devices
        // overlap, the token-rank chain crosses NVLink.  Else: one contiguous shard a device, totals by ncclAllGather.
        if (ctx->peer_ok && total <= ctx->max_bytes && total >= ctx->pipe_min) {
            const int G = static_cast<int>(ctx->devs.size());
            std::vector<std::unique_ptr<LaneLock>> locks(G);
            DeviceCtx* dvs[CFBPE_MAX_DEVICES]; Lane* lns[CFBPE_MAX_DEVICES];
            for (int g = 0; g < G; ++g) {
                dvs[g] = ctx->devs[g].get();
                locks[g].reset(new LaneLock(dvs[g]));
                lns[g] = locks[g]->ln;
                CK(cudaSetDevice(dvs[g]->device));
                rc = wait_for_device_call(ctx, lns[g]);
                if (!rc) rc = ensure_call_buffers(ctx, lns[g], out_starts || chunk, trunc != nullptr, chunk != nullptr, unit && unit->lens);
                if (rc) return rc;
            }
            return run_host_pipelined(ctx, dvs, lns, G, n, bytes, offsets, vocab_ids, out_ids, out_starts, out_cap, out_offsets, out_counts, want_ids, total,
                                      nullptr, nullptr, nullptr, trunc, chunk, unit);
        }
        return run_multi_device(ctx, n, bytes, offsets, vocab_ids, out_ids, out_starts, out_cap, out_offsets, out_counts, want_ids, total, nullptr, trunc,
                                chunk, unit);
    }
    if (total > ctx->max_bytes) return fail(ctx, CFBPE_EINVAL, "batch exceeds max_batch_bytes of this context");
    DeviceCtx* dv = ctx->devs[0].get();
    LaneLock lk(dv);
    return run_lane(ctx, dv, lk.ln, n, bytes, offsets, vocab_ids, out_ids, out_starts, out_cap, out_offsets, out_counts, want_ids, total,
                    nullptr, nullptr, nullptr, trunc, chunk, unit);
}


// A special-token host call on one lane (the whole call on a single-device context, one shard of a multi-device one), as one pass:
// upload, scan (when some vocabulary looks for a special), then the ordinary path on the prompts as they are (no kept match) or
// on the stretches followed by the splice, download.  defer: see run_lane (the results are left in the lane's d_out_* buffers).
int run_lane_special(cfbpe_ctx* ctx, DeviceCtx* dv, Lane* ln, uint32_t n, const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids,
                     const uint8_t* const* modes, uint32_t* out_ids, uint64_t out_cap, uint64_t* out_offsets, uint32_t* out_counts, bool want_ids,
                     uint64_t total, uint32_t* out_bad, uint64_t* defer) {
    CK(cudaSetDevice(dv->device));
    int rc = wait_for_device_call(ctx, ln);
    if (rc) return rc;
    cudaStream_t s = ln->stream.get();
    SpecialSet sp;
    bool scan = false, spliced = false;
    BatchView b;
    if ((rc = special_set(ctx, dv, ln, modes, &sp, &scan, s)) || (rc = upload_batch(ctx, ln, n, bytes, offsets, vocab_ids, total, s, &b))) return rc;
    const EncodeOut plain{want_ids ? ln->d_out_ids.get() : nullptr, ctx->max_bytes, ln->d_out_offsets.get(), ln->d_out_counts.get()};
    const EncodeOut fin{want_ids ? ln->ws.lscratch.rank : nullptr, ctx->max_bytes, ln->sp.fin_offsets.get(), ln->sp.fin_counts.get()};
    if ((rc = enqueue_special_call(ctx, dv, ln, b, sp, scan, s, plain, fin, out_bad, &spliced))) return rc;
    if (spliced) CK(cudaMemcpyAsync(ln->sp.h_status.get(), ln->sp.status.get(), sizeof(SpecialStatus), cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(ln->h_status.get(), ln->ws.status, sizeof(DeviceStatus), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    const DeviceStatus st = *ln->h_status;
    if ((rc = fail_status(ctx, st))) return rc;
    const uint64_t n_tokens = spliced ? ln->sp.h_status->fin.n_tokens : st.n_tokens;
    // where the call's ids, offsets and counts are on the device
    const uint32_t* ids_src = spliced ? ln->ws.lscratch.rank : ln->d_out_ids.get();
    const uint64_t* offs_src = spliced ? ln->sp.fin_offsets.get() : ln->d_out_offsets.get();
    const uint32_t* counts_src = spliced ? ln->sp.fin_counts.get() : ln->d_out_counts.get();
    if (defer) {       // a shard of a multi-device call: its results go where run_multi_device downloads them from
        if (spliced) {
            if (want_ids && n_tokens) CK(cudaMemcpyAsync(ln->d_out_ids.get(), ids_src, n_tokens * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
            CK(cudaMemcpyAsync(ln->d_out_offsets.get(), offs_src, (static_cast<uint64_t>(n) + 1) * sizeof(uint64_t), cudaMemcpyDeviceToDevice, s));
            if (n) CK(cudaMemcpyAsync(ln->d_out_counts.get(), counts_src, static_cast<uint64_t>(n) * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
            CK(cudaStreamSynchronize(s));
        }
        *defer = n_tokens;
        return CFBPE_OK;
    }
    if (out_offsets) CK(cudaMemcpyAsync(out_offsets, offs_src, (static_cast<uint64_t>(n) + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
    if (out_counts && n) CK(cudaMemcpyAsync(out_counts, counts_src, static_cast<uint64_t>(n) * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    if (want_ids && n_tokens > out_cap) {
        CK(cudaStreamSynchronize(s));
        return fail_nospace(ctx, n_tokens, out_offsets, n);
    }
    if (want_ids && n_tokens) CK(cudaMemcpyAsync(out_ids, ids_src, n_tokens * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return CFBPE_OK;
}

// shared body of the special-token host calls
int run_host_special(cfbpe_ctx* ctx, uint32_t n, const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids, const uint8_t* const* modes,
                     uint32_t* out_ids, uint64_t out_cap, uint64_t* out_offsets, uint32_t* out_counts, uint32_t* out_bad) {
    tl_err.clear();
    std::shared_lock<std::shared_mutex> vocabs(ctx->vocab_mu);
    uint64_t total = 0;
    int rc = validate_batch(ctx, n, offsets, vocab_ids, &total);
    if (rc) return rc;
    const bool want_ids = out_ids != nullptr;
    if (total && !bytes) return fail(ctx, CFBPE_EINVAL, "bytes is NULL");
    if (!out_offsets) return fail(ctx, CFBPE_EINVAL, "out_offsets is NULL");
    if (ctx->devs.size() > 1 && n >= ctx->devs.size()) {    // one contiguous shard a device, each with its own special pass
        const SpecialArgs sa{modes, out_bad};
        return run_multi_device(ctx, n, bytes, offsets, vocab_ids, out_ids, nullptr, out_cap, out_offsets, out_counts, want_ids, total, &sa);
    }
    if (total > ctx->max_bytes) return fail(ctx, CFBPE_EINVAL, "batch exceeds max_batch_bytes of this context");
    DeviceCtx* dv = ctx->devs[0].get();
    LaneLock lk(dv);
    return run_lane_special(ctx, dv, lk.ln, n, bytes, offsets, vocab_ids, modes, out_ids, out_cap, out_offsets, out_counts, want_ids, total, out_bad, nullptr);
}

// ---------------------------------------------------------------------------------------
// bytes that are not valid UTF-8 (utf8_repair.cuh)
// ---------------------------------------------------------------------------------------
// the lane's lossy buffers, all or none (as ensure_special_lane).  The caller has selected the lane's device.
int ensure_lossy_lane(cfbpe_ctx* ctx, Lane* ln) {
    if (ln->lossy.h_status) return CFBPE_OK;
    const uint64_t mp = ctx->max_prompts;
    LaneLossy lz;
    bool ok = dmalloc(lz.offsets, mp + 1) == cudaSuccess;
    ok = ok && dmalloc(lz.replaced, mp + 1) == cudaSuccess;
    ok = ok && dmalloc(lz.status, 1) == cudaSuccess;
    ok = ok && hmalloc(lz.h_status, 1) == cudaSuccess;
    if (!ok) { cudaGetLastError(); return fail(ctx, CFBPE_ENOMEM, "no device memory for the lossy-call buffers"); }
    ln->lossy = std::move(lz);
    return CFBPE_OK;
}

// The rest of a lossy call once its batch is on the device: the scan, the one synchronisation of the call (the host needs the
// scan's verdict and the repaired size for the launch geometry), then the ordinary path into `out` on the bytes as they are (no
// invalid byte) or on the repaired batch, which goes to the lane's byte buffer.  When b.bytes IS that buffer (a host call), the
// bytes are first copied to ids_by_pos (4 bytes a byte, dead until the ordinary pass starts).  The prompts' U+FFFD counts are left
// in the lane's replaced buffer.  A repaired batch over max_batch_bytes fails with CFBPE_EINVAL before anything is written to `out`.
int enqueue_lossy_call(cfbpe_ctx* ctx, DeviceCtx* dv, Lane* ln, const BatchView& b, cudaStream_t s, const EncodeOut& out) {
    const LossyWork lw{ln->lossy.replaced.get(), ln->lossy.offsets.get(), ln->lossy.status.get()};
    enqueue_utf8_scan(b, dv->vs, ln->ws, lw, s);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(ln->lossy.h_status.get(), lw.status, sizeof(LossyStatus), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    const LossyScanResult r = lossy_scan_result(*ln->lossy.h_status, b.total_bytes);
    BatchView eb = b;
    if (r.dirty) {
        if (r.total > ctx->max_bytes)
            return fail(ctx, CFBPE_EINVAL, "the repaired batch (" + std::to_string(r.total) + " bytes) exceeds max_batch_bytes of this context");
        BatchView raw = b;
        if (b.bytes == ln->d_bytes.get()) {
            uint8_t* stage = reinterpret_cast<uint8_t*>(ln->ws.ids_by_pos);
            CK(cudaMemcpyAsync(stage, b.bytes, b.total_bytes, cudaMemcpyDeviceToDevice, s));
            raw.bytes = stage;
        }
        enqueue_utf8_repair(raw, ln->ws, lw, ln->d_bytes.get(), r.total, s);
        eb = BatchView{ln->d_bytes.get(), lw.offsets, b.vocab_ids, b.n_prompts, r.total};
    }
    enqueue_encode(eb, dv->vs, dv->uc, ln->ws, out.ids, out.cap, out.offsets, out.counts, static_cast<uint32_t>(dv->sm_count * 4),
                   s, ln->aux_stream.get(), ln->aux2_stream.get(), ln->ev_fork.get(), ln->ev_join.get(), ln->ev_join2.get(), static_cast<ProfEvents*>(nullptr));
    CK(cudaGetLastError());
    return CFBPE_OK;
}

// A lossy host call on one lane (the whole call on a single-device context, one shard of a multi-device one), as one pass: upload,
// scan, the ordinary path on the prompts as they are or repaired, download.  defer: see run_lane (the ids, offsets and counts are
// left in the lane's d_out_* buffers, the U+FFFD counts in its replaced buffer).
int run_lane_lossy(cfbpe_ctx* ctx, DeviceCtx* dv, Lane* ln, uint32_t n, const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids,
                   uint32_t* out_ids, uint64_t out_cap, uint64_t* out_offsets, uint32_t* out_counts, bool want_ids, uint64_t total,
                   uint32_t* out_replaced, uint64_t* defer) {
    CK(cudaSetDevice(dv->device));
    int rc = wait_for_device_call(ctx, ln);
    if (!rc) rc = ensure_lossy_lane(ctx, ln);
    if (rc) return rc;
    cudaStream_t s = ln->stream.get();
    BatchView b;
    if ((rc = upload_batch(ctx, ln, n, bytes, offsets, vocab_ids, total, s, &b))) return rc;
    const EncodeOut out{want_ids ? ln->d_out_ids.get() : nullptr, ctx->max_bytes, ln->d_out_offsets.get(), ln->d_out_counts.get()};
    if ((rc = enqueue_lossy_call(ctx, dv, ln, b, s, out))) return rc;
    CK(cudaMemcpyAsync(ln->h_status.get(), ln->ws.status, sizeof(DeviceStatus), cudaMemcpyDeviceToHost, s));
    if (!defer) {
        if (out_offsets) CK(cudaMemcpyAsync(out_offsets, ln->d_out_offsets.get(), (static_cast<uint64_t>(n) + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
        if (out_counts && n) CK(cudaMemcpyAsync(out_counts, ln->d_out_counts.get(), static_cast<uint64_t>(n) * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        if (out_replaced && n) CK(cudaMemcpyAsync(out_replaced, ln->lossy.replaced.get(), static_cast<uint64_t>(n) * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    }
    CK(cudaStreamSynchronize(s));
    const DeviceStatus st = *ln->h_status;
    if ((rc = fail_status(ctx, st))) return rc;
    if (defer) { *defer = st.n_tokens; return CFBPE_OK; }
    if (want_ids && st.n_tokens > out_cap) return fail_nospace(ctx, st.n_tokens, out_offsets, n);
    if (want_ids && st.n_tokens) {
        CK(cudaMemcpyAsync(out_ids, ln->d_out_ids.get(), st.n_tokens * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        CK(cudaStreamSynchronize(s));
    }
    return CFBPE_OK;
}

// shared body of the lossy host call
int run_host_lossy(cfbpe_ctx* ctx, uint32_t n, const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids, uint32_t* out_ids,
                   uint64_t out_cap, uint64_t* out_offsets, uint32_t* out_counts, uint32_t* out_replaced) {
    tl_err.clear();
    std::shared_lock<std::shared_mutex> vocabs(ctx->vocab_mu);
    uint64_t total = 0;
    int rc = validate_batch(ctx, n, offsets, vocab_ids, &total);
    if (rc) return rc;
    const bool want_ids = out_ids != nullptr;
    if (total && !bytes) return fail(ctx, CFBPE_EINVAL, "bytes is NULL");
    if (!out_offsets) return fail(ctx, CFBPE_EINVAL, "out_offsets is NULL");
    if (ctx->devs.size() > 1 && n >= ctx->devs.size()) {    // one contiguous shard a device, each with its own scan and repair
        const LossyArgs la{out_replaced};
        return run_multi_device(ctx, n, bytes, offsets, vocab_ids, out_ids, nullptr, out_cap, out_offsets, out_counts, want_ids, total, nullptr,
                                nullptr, nullptr, nullptr, &la);
    }
    if (total > ctx->max_bytes) return fail(ctx, CFBPE_EINVAL, "batch exceeds max_batch_bytes of this context");
    DeviceCtx* dv = ctx->devs[0].get();
    LaneLock lk(dv);
    return run_lane_lossy(ctx, dv, lk.ln, n, bytes, offsets, vocab_ids, out_ids, out_cap, out_offsets, out_counts, want_ids, total, out_replaced, nullptr);
}

// ---------------------------------------------------------------------------------------
// construction / destruction
// ---------------------------------------------------------------------------------------
// everything one call touches on the device, sized by max_batch_bytes (~33 bytes per byte of it)
bool create_lane(Lane* ln, int device, uint64_t mb, uint64_t mp) {
    ln->device = device;
    ln->max_bytes = mb;
    int prio_lo = 0, prio_hi = 0;
    cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
    bool ok = make_stream(ln->stream, prio_hi) == cudaSuccess;   // front stream of sub-batch 0
    ok = ok && dmalloc(ln->d_bytes, lane_bytes_alloc(mb, kMaxPipeChunks)) == cudaSuccess;
    ok = ok && dmalloc(ln->d_offsets, lane_offsets_alloc(mp, kMaxPipeChunks)) == cudaSuccess;
    ok = ok && dmalloc(ln->d_vocab_ids, mp + 1) == cudaSuccess;
    ok = ok && dmalloc(ln->d_out_ids, mb + 1) == cudaSuccess;
    ok = ok && dmalloc(ln->d_out_offsets, lane_offsets_alloc(mp, kMaxPipeChunks)) == cudaSuccess;
    ok = ok && dmalloc(ln->d_out_counts, mp + 1) == cudaSuccess;
    const WsSizes ws = workspace_alloc(mb, kMaxPipeChunks);
    for_each_ws_buffer(ln->ws, [&](auto*& p, WsKind kind) { ok = ok && dmalloc(&p, ws.n[kind]) == cudaSuccess; });
    set_workspace_caps(ln->ws, ws);      // a one-shot call may use all of it
    ok = ok && dmalloc(ln->d_dec_sums, mb / kDecodeTile + 2) == cudaSuccess;
    ok = ok && dmalloc(ln->d_dec_base, mb / kDecodeTile + 2) == cudaSuccess;
    ok = ok && dmalloc(ln->d_totals, CFBPE_MAX_DEVICES + 1) == cudaSuccess;
    ok = ok && dmalloc(ln->d_status, 1) == cudaSuccess;
    ln->ws.status = ln->d_status.get();
    ok = ok && hmalloc(ln->h_status, 1) == cudaSuccess;
    ok = ok && hmalloc(ln->h_totals, CFBPE_MAX_DEVICES + 1) == cudaSuccess;
    ok = ok && make_stream(ln->h2d_stream, 0) == cudaSuccess;      // (0: the default priority)
    ok = ok && make_stream(ln->d2h_stream, 0) == cudaSuccess;
    ok = ok && dmalloc(ln->d_status_arr, kMaxPipeChunks) == cudaSuccess;
    ok = ok && hmalloc(ln->h_status_arr, kMaxPipeChunks) == cudaSuccess;
    ok = ok && hmalloc(ln->h_offs_stage, lane_offsets_alloc(mp, kMaxPipeChunks)) == cudaSuccess;
    {   // a pipelined host call gives earlier sub-batches the higher priority, so that they finish first and their downloads
        // run while the later ones compute (with equal priorities the sub-batches finished together and the downloads queued up
        // at the end: tools/pipe_trace.py)
        const int levels = prio_lo - prio_hi + 1;
        for (int k = 1; ok && k < kFrontStreams; ++k) ok = make_stream(ln->front[k], prio_hi + (k < levels ? k : levels - 1)) == cudaSuccess;
        for (int k = 0; ok && k < kSideStreams; ++k) ok = make_stream(ln->side[k], prio_hi) == cudaSuccess;
        for (int k = 0; ok && k < kSideStreams; ++k) ok = make_stream(ln->side2[k], prio_hi) == cudaSuccess;
        if (const char* e = std::getenv("CFBPE_PIPE_PRIO")) {      // experiment: 1 = every kernel at one priority, 2 = priority by the sub-batch's age
            ln->prio_mode = std::atoi(e);
            ln->prio_levels = ln->prio_mode == 2 ? (levels < kPrioLevels ? levels : kPrioLevels) : 1;
            for (int l = 0; ok && ln->prio_mode && l < ln->prio_levels; ++l)
                for (int j = 0; ok && j < kPoolSlots; ++j) ok = make_stream(ln->pool[l][j], prio_hi + l) == cudaSuccess;
        }
    }
    // the long-piece kernels are latency-bound and small: their CTAs go first, the short-piece kernels fill the rest
    // (A/B of lower priorities and of CTA caps: no gain)
    ok = ok && make_stream(ln->aux_stream, prio_hi) == cudaSuccess;
    ok = ok && make_stream(ln->aux2_stream, prio_hi) == cudaSuccess;
    ok = ok && make_event(ln->ev_fork, cudaEventDisableTiming) == cudaSuccess && make_event(ln->ev_join, cudaEventDisableTiming) == cudaSuccess;
    ok = ok && make_event(ln->ev_ws, cudaEventDisableTiming) == cudaSuccess;
    ok = ok && make_event(ln->ev_join2, cudaEventDisableTiming) == cudaSuccess;
    for (int k = 0; ok && k < kMaxPipeChunks; ++k)
        ok = make_event(ln->ev_h2d[k], cudaEventDisableTiming) == cudaSuccess && make_event(ln->ev_front[k], cudaEventDisableTiming) == cudaSuccess &&
             make_event(ln->ev_done[k], cudaEventDisableTiming) == cudaSuccess && make_event(ln->ev_chain[k], cudaEventDisableTiming) == cudaSuccess &&
             make_event(ln->ev_scan[k], cudaEventDisableTiming) == cudaSuccess && make_event(ln->ev_list[k], cudaEventDisableTiming) == cudaSuccess;
    ok = ok && cudaMemset(ln->d_bytes.get(), 0, lane_bytes_alloc(mb, kMaxPipeChunks)) == cudaSuccess;
    for (int k = 0; ok && k < CFBPE_NUM_KERNELS; ++k)
        ok = make_event(ln->prof.ev[k][0], cudaEventDefault) == cudaSuccess && make_event(ln->prof.ev[k][1], cudaEventDefault) == cudaSuccess;
    for (int k = 0; ok && k < 2; ++k)
        ok = make_event(ln->prof.h2d[k], cudaEventDefault) == cudaSuccess && make_event(ln->prof.d2h[k], cudaEventDefault) == cudaSuccess &&
             make_event(ln->prof.total[k], cudaEventDefault) == cudaSuccess;
    return ok;
}

bool create_device(DeviceCtx* dv, int device, int index, uint32_t n_lanes, uint64_t mb, uint64_t mp) {
    dv->device = device; dv->index = index;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess || prop.major != 9 || prop.minor != 0) return false;     // sm_90a SASS only
    if (cudaSetDevice(device) != cudaSuccess) return false;
    dv->sm_count = prop.multiProcessorCount;
    bool ok = cudaFuncSetAttribute(bpe_list_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kListSmemBytes)) == cudaSuccess;
    ok = ok && cudaFuncSetAttribute(pretok_split16_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kNumPatterns * kProdTableBytes)) == cudaSuccess;
    ok = ok && dmalloc(dv->d_uc1, sizeof cfbpe_uc_stage1) == cudaSuccess;
    ok = ok && dmalloc(dv->d_uc2, sizeof cfbpe_uc_stage2) == cudaSuccess;
    ok = ok && cudaMemcpy(dv->d_uc1.get(), cfbpe_uc_stage1, sizeof cfbpe_uc_stage1, cudaMemcpyHostToDevice) == cudaSuccess;
    ok = ok && cudaMemcpy(dv->d_uc2.get(), cfbpe_uc_stage2, sizeof cfbpe_uc_stage2, cudaMemcpyHostToDevice) == cudaSuccess;
    {
        std::vector<uint16_t> fsm(kNumPatterns * kPretokTableSize);
        uint8_t ascii[128];
        build_pretok_tables(fsm.data());
        build_ascii_classes(ascii);
        ok = ok && dmalloc(dv->d_ascii, 128) == cudaSuccess;
        ok = ok && dmalloc(dv->d_fsm, fsm.size()) == cudaSuccess;
        ok = ok && cudaMemcpy(dv->d_ascii.get(), ascii, 128, cudaMemcpyHostToDevice) == cudaSuccess;
        ok = ok && cudaMemcpy(dv->d_fsm.get(), fsm.data(), fsm.size() * sizeof(uint16_t), cudaMemcpyHostToDevice) == cudaSuccess;
        std::vector<SplitTablesHost> st(1);
        build_split_tables(st.data());
        ok = ok && dmalloc(dv->d_split_tables, sizeof(SplitTablesHost)) == cudaSuccess;
        ok = ok && cudaMemcpy(dv->d_split_tables.get(), st.data(), sizeof(SplitTablesHost), cudaMemcpyHostToDevice) == cudaSuccess;
    }
    if (!ok) return false;
    dv->uc = UcTables{dv->d_uc1.get(), dv->d_uc2.get(), dv->d_ascii.get(), dv->d_fsm.get(),
                      dv->d_split_tables.get() + offsetof(SplitTablesHost, cls256),
                      reinterpret_cast<const uint16_t*>(dv->d_split_tables.get() + offsetof(SplitTablesHost, fsm16)),
                      reinterpret_cast<const uint16_t*>(dv->d_split_tables.get() + offsetof(SplitTablesHost, ctx16)),
                      reinterpret_cast<const uint64_t*>(dv->d_split_tables.get() + offsetof(SplitTablesHost, prod)),
                      reinterpret_cast<const ProdInfo*>(dv->d_split_tables.get() + offsetof(SplitTablesHost, prod_info)),
                      dv->d_split_tables.get() + offsetof(SplitTablesHost, prod_skip),
                      dv->d_split_tables.get() + offsetof(SplitTablesHost, prod_start)};
    for (uint32_t i = 0; i < n_lanes; ++i) {
        dv->lanes.emplace_back(new Lane());
        if (!create_lane(dv->lanes.back().get(), device, mb, mp)) return false;
    }
    return true;
}

bool load_nccl(NcclApi* n) {
    for (const char* name : {"libnccl.so.2", "libnccl.so"}) { n->lib = dlopen(name, RTLD_NOW | RTLD_GLOBAL); if (n->lib) break; }
    if (!n->lib) return false;
    auto sym = [&](const char* s) { return dlsym(n->lib, s); };
    n->CommInitAll = reinterpret_cast<decltype(n->CommInitAll)>(sym("ncclCommInitAll"));
    n->CommDestroy = reinterpret_cast<decltype(n->CommDestroy)>(sym("ncclCommDestroy"));
    n->GroupStart = reinterpret_cast<decltype(n->GroupStart)>(sym("ncclGroupStart"));
    n->GroupEnd = reinterpret_cast<decltype(n->GroupEnd)>(sym("ncclGroupEnd"));
    n->Broadcast = reinterpret_cast<decltype(n->Broadcast)>(sym("ncclBroadcast"));
    n->AllGather = reinterpret_cast<decltype(n->AllGather)>(sym("ncclAllGather"));
    n->GetErrorString = reinterpret_cast<decltype(n->GetErrorString)>(sym("ncclGetErrorString"));
    return n->CommInitAll && n->CommDestroy && n->GroupStart && n->GroupEnd && n->Broadcast && n->AllGather && n->GetErrorString;
}

// what the lane's last device-path call reports, once its status is in h_status: the status, then ENOSPC against its out_cap
int device_call_status(cfbpe_ctx* ctx, const Lane* ln) {
    const DeviceStatus& st = *ln->h_status;
    if (const int rc = fail_status(ctx, st)) return rc;
    if (ln->dev_want_ids && st.n_tokens > ln->dev_out_cap) return fail_nospace(ctx, st.n_tokens);
    return CFBPE_OK;
}

// The shape of a device-path call (the caller's device buffers, the caller's stream): the checks (d_out: the call's required output);
// the device of the buffers (the
// first of the context whose ordinal is current, else the first) and a lane of it; the stream ordered after the lane's previous
// device-path call; then enqueue(dv, ln, b, s, prof) queues the work (prof: profiling, when `profiled` and the context profiles).
// The lane's workspace stays busy until that has run (ev_ws).  With n_tokens or profiling the call waits and reports the status.
template <typename F>
int device_call(cfbpe_ctx* ctx, uint32_t n_prompts, const uint8_t* d_bytes, uint64_t total_bytes, const uint64_t* d_offsets,
                const uint8_t* d_vocab_ids, const void* d_out, bool want_ids, uint64_t out_cap, uint64_t* n_tokens, void* stream,
                bool profiled, F&& enqueue) {
    std::shared_lock<std::shared_mutex> vocabs(ctx->vocab_mu);
    if (n_prompts > ctx->max_prompts || total_bytes > ctx->max_bytes) return fail(ctx, CFBPE_EINVAL, "batch exceeds the limits of this context");
    if (!d_offsets || !d_out || (total_bytes && !d_bytes)) return fail(ctx, CFBPE_EINVAL, "device pointer is NULL");
    if (!ctx->vocabs[0].loaded && !d_vocab_ids) return fail(ctx, CFBPE_ENOENT, "vocab 0 is not loaded");
    if (!ctx->loaded_mask) return fail(ctx, CFBPE_ENOENT, "no vocabulary is loaded");
    DeviceCtx* dv = ctx->devs[0].get();
    { int cur = -1; if (cudaGetDevice(&cur) == cudaSuccess) for (auto& d : ctx->devs) if (d->device == cur) dv = d.get(); }
    LaneLock lk(dv);
    Lane* ln = lk.ln;
    CK(cudaSetDevice(dv->device));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    // a lane is one workspace: a call on another stream waits (on the device) for the lane's previous device-path call;
    // consecutive calls take different lanes when the context has several (n_workspaces) and then overlap
    if (ln->ws_pending) CK(cudaStreamWaitEvent(s, ln->ev_ws.get(), 0));
    ProfEvents* prof = profiled && ctx->profiling.load() ? &ln->prof : nullptr;
    if (prof) { std::memset(prof->launched, 0, sizeof prof->launched); cudaEventRecord(prof->total[0].get(), s); cudaEventRecord(prof->h2d[0].get(), s); cudaEventRecord(prof->h2d[1].get(), s); }
    const int rc = enqueue(dv, ln, BatchView{d_bytes, d_offsets, d_vocab_ids, n_prompts, total_bytes}, s, prof);
    if (rc) return rc;
    CK(cudaEventRecord(ln->ev_ws.get(), s));
    ln->ws_pending = true;
    ln->dev_out_cap = out_cap;
    ln->dev_want_ids = want_ids;
    tl_device_lane = ln;
    if (prof) { cudaEventRecord(prof->d2h[0].get(), s); cudaEventRecord(prof->d2h[1].get(), s); cudaEventRecord(prof->total[1].get(), s); }
    if (!n_tokens && !prof) return CFBPE_OK;
    CK(cudaMemcpyAsync(ln->h_status.get(), ln->ws.status, sizeof(DeviceStatus), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    if (prof) fill_profile(ln, total_bytes);
    if (n_tokens) *n_tokens = ln->h_status->n_tokens;
    return device_call_status(ctx, ln);
}

// shared body of encode_batch_device / encode_batch_starts_device / encode_batch_char_starts_device: d_out_starts (nullable) gets the
// starts, beside d_out_ids; unit (nullable): in code points or UTF-16 units, and the prompts' lengths in them
int run_device(cfbpe_ctx* ctx, uint32_t n_prompts, const uint8_t* d_bytes, uint64_t total_bytes, const uint64_t* d_offsets,
               const uint8_t* d_vocab_ids, uint32_t* d_out_ids, uint32_t* d_out_starts, uint64_t out_cap, uint64_t* d_out_offsets,
               uint32_t* d_out_counts, uint64_t* n_tokens, void* stream, const UnitView* unit = nullptr) {
    return device_call(ctx, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, d_out_offsets, d_out_ids != nullptr, out_cap, n_tokens, stream, true,
                       [&](DeviceCtx* dv, Lane* ln, const BatchView& b, cudaStream_t s, ProfEvents* prof) {
        enqueue_encode(b, dv->vs, dv->uc, ln->ws, d_out_ids, out_cap, d_out_offsets, d_out_counts,
                       static_cast<uint32_t>(dv->sm_count * 4), s, prof ? s : ln->aux_stream.get(), prof ? s : ln->aux2_stream.get(),
                       ln->ev_fork.get(), ln->ev_join.get(), ln->ev_join2.get(), prof, nullptr, d_out_starts, nullptr, nullptr,
                       unit);   // profiling: one stream, so that the per-kernel times do not overlap
        CK(cudaGetLastError());
        return CFBPE_OK;
    });
}

// shared body of encode_batch_special_device
int run_device_special(cfbpe_ctx* ctx, uint32_t n_prompts, const uint8_t* d_bytes, uint64_t total_bytes, const uint64_t* d_offsets,
                       const uint8_t* d_vocab_ids, const uint8_t* const* modes, uint32_t* d_out_ids, uint64_t out_cap, uint64_t* d_out_offsets,
                       uint32_t* d_out_counts, uint64_t* n_tokens, uint32_t* out_bad, void* stream) {
    return device_call(ctx, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, d_out_offsets, d_out_ids != nullptr, out_cap, n_tokens, stream, false,
                       [&](DeviceCtx* dv, Lane* ln, const BatchView& b, cudaStream_t s, ProfEvents*) {
        SpecialSet sp;
        bool scan = false, spliced = false;
        const EncodeOut out{d_out_ids, out_cap, d_out_offsets, d_out_counts};
        int rc = special_set(ctx, dv, ln, modes, &sp, &scan, s);
        if (!rc) rc = enqueue_special_call(ctx, dv, ln, b, sp, scan, s, out, out, out_bad, &spliced);
        // the lane's status carries the call's id count (cfbpe_device_status checks it against out_cap): n_tokens and tok_end
        if (!rc && spliced) CK(cudaMemcpyAsync(&ln->ws.status->n_tokens, &ln->sp.status->fin.n_tokens, 2 * sizeof(uint64_t), cudaMemcpyDeviceToDevice, s));
        return rc;
    });
}

// shared body of encode_batch_lossy_device: the repaired batch (when one is needed) goes to the lane's byte buffer; the U+FFFD counts
// are copied to d_out_replaced once the repaired size is known to fit
int run_device_lossy(cfbpe_ctx* ctx, uint32_t n_prompts, const uint8_t* d_bytes, uint64_t total_bytes, const uint64_t* d_offsets,
                     const uint8_t* d_vocab_ids, uint32_t* d_out_ids, uint64_t out_cap, uint64_t* d_out_offsets, uint32_t* d_out_counts,
                     uint32_t* d_out_replaced, uint64_t* n_tokens, void* stream) {
    return device_call(ctx, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, d_out_offsets, d_out_ids != nullptr, out_cap, n_tokens, stream, false,
                       [&](DeviceCtx* dv, Lane* ln, const BatchView& b, cudaStream_t s, ProfEvents*) {
        int rc = ensure_lossy_lane(ctx, ln);
        if (!rc) rc = enqueue_lossy_call(ctx, dv, ln, b, s, EncodeOut{d_out_ids, out_cap, d_out_offsets, d_out_counts});
        if (!rc && d_out_replaced && n_prompts)
            CK(cudaMemcpyAsync(d_out_replaced, ln->lossy.replaced.get(), static_cast<uint64_t>(n_prompts) * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
        return rc;
    });
}

// shared body of truncate_batch_device: the ids and offsets go to the lane's buffers (max_batch_bytes ids fit: no ENOSPC)
int run_device_truncate(cfbpe_ctx* ctx, uint32_t n_prompts, const uint8_t* d_bytes, uint64_t total_bytes, const uint64_t* d_offsets,
                        const uint8_t* d_vocab_ids, const uint32_t* d_budgets, uint32_t mode, uint32_t* d_out_cut, uint32_t* d_out_kept,
                        uint32_t* d_out_counts, void* stream) {
    return device_call(ctx, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, d_out_cut, false, 0, nullptr, stream, true,
                       [&](DeviceCtx* dv, Lane* ln, const BatchView& b, cudaStream_t s, ProfEvents* prof) {
        const TruncateView tv{d_budgets, mode == CFBPE_TRUNCATE_TAIL ? 1u : 0u, d_out_cut, d_out_kept};
        enqueue_encode(b, dv->vs, dv->uc, ln->ws, ln->d_out_ids.get(), ctx->max_bytes, ln->d_out_offsets.get(), d_out_counts,
                       static_cast<uint32_t>(dv->sm_count * 4), s, prof ? s : ln->aux_stream.get(), prof ? s : ln->aux2_stream.get(),
                       ln->ev_fork.get(), ln->ev_join.get(), ln->ev_join2.get(), prof, nullptr, nullptr, &tv);
        CK(cudaGetLastError());
        return CFBPE_OK;
    });
}

// shared body of chunk_batch_device: the ids, offsets and starts go to the lane's buffers (max_batch_bytes ids fit); the status
// carries the chunk count where device_call and cfbpe_device_status look for the id count, so ENOSPC is checked against chunk_cap
int run_device_chunk(cfbpe_ctx* ctx, uint32_t n_prompts, const uint8_t* d_bytes, uint64_t total_bytes, const uint64_t* d_offsets,
                     const uint8_t* d_vocab_ids, uint32_t chunk_tokens, uint32_t overlap_tokens, uint32_t* d_out_spans, uint64_t chunk_cap,
                     uint64_t* d_out_chunk_offsets, uint32_t* d_out_counts, uint64_t* n_chunks, void* stream) {
    return device_call(ctx, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, d_out_chunk_offsets, true, chunk_cap, n_chunks, stream, true,
                       [&](DeviceCtx* dv, Lane* ln, const BatchView& b, cudaStream_t s, ProfEvents* prof) {
        if (const int rc = ensure_call_buffers(ctx, ln, true, false, false)) return rc;     // the starts
        const ChunkView cv{chunk_tokens, chunk_tokens - overlap_tokens, d_out_chunk_offsets, nullptr, d_out_spans, d_out_spans + 1, 2u, chunk_cap};
        enqueue_encode(b, dv->vs, dv->uc, ln->ws, ln->d_out_ids.get(), ctx->max_bytes, ln->d_out_offsets.get(), d_out_counts,
                       static_cast<uint32_t>(dv->sm_count * 4), s, prof ? s : ln->aux_stream.get(), prof ? s : ln->aux2_stream.get(),
                       ln->ev_fork.get(), ln->ev_join.get(), ln->ev_join2.get(), prof, nullptr, ln->d_out_starts.get(), nullptr, &cv);
        CK(cudaGetLastError());
        static_assert(offsetof(DeviceStatus, chunk_end) == offsetof(DeviceStatus, n_chunks) + sizeof(uint64_t) &&
                      offsetof(DeviceStatus, tok_end) == offsetof(DeviceStatus, n_tokens) + sizeof(uint64_t), "count, then end");
        CK(cudaMemcpyAsync(&ln->ws.status->n_tokens, &ln->ws.status->n_chunks, 2 * sizeof(uint64_t), cudaMemcpyDeviceToDevice, s));
        return CFBPE_OK;
    });
}

}  // namespace

// Every entry point that selects a device puts the caller's current device back on return: the library is a guest in the host
// process (a model runtime next door expects its own device to stay current on its thread).
struct DeviceGuard {
    int prev = -1;
    DeviceGuard() { if (cudaGetDevice(&prev) != cudaSuccess) { prev = -1; cudaGetLastError(); } }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

extern "C" {

int cfbpe_abi_version(void) { return static_cast<int>(CFBPE_ABI_VERSION); }

#ifndef CFBPE_SRC_HASH
#define CFBPE_SRC_HASH "unknown"
#endif
const char* cfbpe_build_id(void) { return CFBPE_SRC_HASH; }

int cfbpe_create(const cfbpe_config* cfg, cfbpe_ctx** out) {
    DeviceGuard restore_device;
    if (!cfg || !out || cfg->struct_size < offsetof(cfbpe_config, devices)) return CFBPE_EINVAL;
    *out = nullptr;
    // (a pipelined host call keeps ~20 streams busy: hosts should export CUDA_DEVICE_MAX_CONNECTIONS=32 before CUDA
    //  initialises -- INTEGRATION.md; the library does not touch the process environment)
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return CFBPE_ENODEV;
    // the fields after `flags` exist when the caller's struct is new enough (struct_size versions the struct)
    const bool has_multi = cfg->struct_size >= sizeof(cfbpe_config);
    std::vector<int> devices;
    if (has_multi && cfg->n_devices > 0) {
        if (cfg->n_devices > CFBPE_MAX_DEVICES) return CFBPE_EINVAL;
        for (uint32_t i = 0; i < cfg->n_devices; ++i) devices.push_back(cfg->devices[i]);
    } else devices.push_back(cfg->device);
    for (size_t i = 0; i < devices.size(); ++i) {
        if (devices[i] < 0 || devices[i] >= ndev) return CFBPE_ENODEV;
        for (size_t j = 0; j < i; ++j) if (devices[j] == devices[i]) return CFBPE_EINVAL;
    }
    cfbpe_ctx* ctx = new (std::nothrow) cfbpe_ctx();
    if (!ctx) return CFBPE_ENOMEM;
    ctx->max_bytes = cfg->max_batch_bytes ? cfg->max_batch_bytes : (256ull << 20);
    ctx->max_prompts = cfg->max_prompts ? cfg->max_prompts : (1u << 20);
    ctx->n_workspaces = (has_multi && cfg->n_workspaces) ? cfg->n_workspaces : 1u;
    if (ctx->max_bytes >= (1ull << 32) - 4096 || ctx->n_workspaces > 16) { delete ctx; return CFBPE_EINVAL; }   // byte positions inside a batch are 32-bit in the work lists
    if (devices.size() > 1 && !load_nccl(&ctx->nccl)) { delete ctx; tl_err = "a multi-device context needs libnccl.so.2 (vocabulary broadcast, gather of the shard totals)"; return CFBPE_EIO; }
    for (size_t i = 0; i < devices.size(); ++i) {
        ctx->devs.emplace_back(new DeviceCtx());
        if (!create_device(ctx->devs.back().get(), devices[i], static_cast<int>(i), ctx->n_workspaces, ctx->max_bytes, ctx->max_prompts)) {
            const bool nodev = ctx->devs.back()->sm_count == 0;     // refused before anything was allocated: not an sm_90 device
            cudaGetLastError();
            cfbpe_destroy(ctx);
            return nodev ? CFBPE_ENODEV : CFBPE_ENOMEM;
        }
    }
    if (devices.size() > 1) {
        std::vector<void*> comms(devices.size(), nullptr);
        const int rc = ctx->nccl.CommInitAll(comms.data(), static_cast<int>(devices.size()), devices.data());
        if (rc != 0) { tl_err = std::string("ncclCommInitAll: ") + ctx->nccl.GetErrorString(rc); cfbpe_destroy(ctx); return CFBPE_EIO; }
        for (size_t i = 0; i < devices.size(); ++i) ctx->devs[i]->comm = comms[i];
        // peer mappings: a sub-batch on one device reads the token rank its predecessor on another device ended at
        bool peers = std::getenv("CFBPE_NO_PEER") == nullptr;
        for (size_t a = 0; a < devices.size() && peers; ++a) {
            cudaSetDevice(devices[a]);
            for (size_t b2 = 0; b2 < devices.size() && peers; ++b2) {
                if (a == b2) continue;
                int can = 0;
                if (cudaDeviceCanAccessPeer(&can, devices[a], devices[b2]) != cudaSuccess || !can) { peers = false; break; }
                const cudaError_t e = cudaDeviceEnablePeerAccess(devices[b2], 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) peers = false;
                cudaGetLastError();
            }
        }
        ctx->peer_ok = peers;
    }
    if (const char* e = std::getenv("CFBPE_PIPE_CHUNK_BYTES")) { const uint64_t v = std::strtoull(e, nullptr, 10); if (v >= 1024) ctx->pipe_chunk = v; }
    if (const char* e = std::getenv("CFBPE_PIPE_MIN_BYTES")) { const uint64_t v = std::strtoull(e, nullptr, 10); if (v >= 1) ctx->pipe_min = v; }
    *out = ctx;
    return CFBPE_OK;
}

void cfbpe_destroy(cfbpe_ctx* ctx) {
    DeviceGuard restore_device;
    if (!ctx) return;
    for (auto& dv : ctx->devs) {
        cudaSetDevice(dv->device);
        cudaDeviceSynchronize();             // device-path calls may still be running on the caller's streams
        if (dv->comm && ctx->nccl.CommDestroy) ctx->nccl.CommDestroy(dv->comm);
        dv.reset();                          // its lanes, then its tables
    }
    delete ctx;
}

const char* cfbpe_last_error(const cfbpe_ctx*) { return tl_err.c_str(); }

int cfbpe_vocab_load(cfbpe_ctx* ctx, uint32_t vocab_id, const uint8_t* ranks_file, size_t len, uint32_t format,
                     uint32_t pattern_id, uint32_t max_ranks) {
    DeviceGuard restore_device;
    if (!ctx) return CFBPE_EINVAL;
    tl_err.clear();
    if (vocab_id >= CFBPE_MAX_VOCABS) return fail(ctx, CFBPE_EINVAL, "vocab_id out of range");
    if (!ranks_file || !len) return fail(ctx, CFBPE_EINVAL, "empty rank file");
    if (pattern_id >= CFBPE_PATTERN_COUNT) return fail(ctx, CFBPE_EINVAL, "unknown pattern id");
    std::vector<std::string> toks;
    std::string e;
    int rc;
    if (format == CFBPE_FORMAT_TIKTOKEN) rc = parse_tiktoken(ranks_file, len, max_ranks, toks, e);
    else if (format == CFBPE_FORMAT_TEKKEN_JSON) rc = parse_tekken_json(ranks_file, len, max_ranks, toks, e);
    else return fail(ctx, CFBPE_EINVAL, "unknown rank-file format");
    if (rc) return fail(ctx, rc, e);
    std::vector<uint8_t> blob;
    rc = build_tables(toks, pattern_id, blob, e);
    if (rc) return fail(ctx, rc, e);
    std::unique_lock<std::shared_mutex> lock(ctx->vocab_mu);
    return install_blob(ctx, vocab_id, std::move(blob));
}

int cfbpe_vocab_get_info(const cfbpe_ctx* ctx, uint32_t vocab_id, cfbpe_vocab_info* out) {
    if (!ctx || !out || vocab_id >= CFBPE_MAX_VOCABS) return CFBPE_EINVAL;
    const HostVocab& v = ctx->vocabs[vocab_id];
    if (!v.loaded) return CFBPE_ENOENT;
    out->n_ranks = v.hdr.n_ranks;
    out->pattern_id = v.hdr.pattern_id;
    out->max_token_len = v.hdr.max_token_len;
    out->n_pair_entries = v.hdr.n_pair_entries;
    out->table_bytes = v.hdr.total_bytes;
    return CFBPE_OK;
}

int cfbpe_vocab_export(const cfbpe_ctx* ctx, uint32_t vocab_id, uint8_t* buf, uint64_t cap, uint64_t* size) {
    if (!ctx || vocab_id >= CFBPE_MAX_VOCABS) return CFBPE_EINVAL;
    const HostVocab& v = ctx->vocabs[vocab_id];
    if (!v.loaded) return CFBPE_ENOENT;
    if (size) *size = v.h_blob.size();
    if (!buf) return CFBPE_OK;
    if (cap < v.h_blob.size()) return CFBPE_ENOSPC;
    std::memcpy(buf, v.h_blob.data(), v.h_blob.size());
    return CFBPE_OK;
}

int cfbpe_vocab_import(cfbpe_ctx* ctx, uint32_t vocab_id, const uint8_t* buf, uint64_t size) {
    DeviceGuard restore_device;
    if (!ctx) return CFBPE_EINVAL;
    tl_err.clear();
    if (vocab_id >= CFBPE_MAX_VOCABS || !buf) return fail(ctx, CFBPE_EINVAL, "bad argument");
    std::string e;
    int rc = validate_tables(buf, size, e);
    if (rc) return fail(ctx, rc, e);
    std::unique_lock<std::shared_mutex> lock(ctx->vocab_mu);
    return install_blob(ctx, vocab_id, std::vector<uint8_t>(buf, buf + size));
}

int cfbpe_encode_batch(cfbpe_ctx* ctx, uint32_t n_prompts, const uint8_t* bytes, const uint64_t* offsets,
                       const uint8_t* vocab_ids, uint32_t* out_ids, uint64_t out_cap, uint64_t* out_offsets,
                       uint32_t* out_counts) {
    DeviceGuard restore_device;
    if (!ctx) return CFBPE_EINVAL;
    return run_host(ctx, n_prompts, bytes, offsets, vocab_ids, out_ids, nullptr, out_cap, out_offsets, out_counts, true);
}

int cfbpe_encode_batch_starts(cfbpe_ctx* ctx, uint32_t n_prompts, const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids,
                              uint32_t* out_ids, uint32_t* out_starts, uint64_t out_cap, uint64_t* out_offsets, uint32_t* out_counts) {
    DeviceGuard restore_device;
    if (!ctx) return CFBPE_EINVAL;
    tl_err.clear();
    if (!out_ids || !out_starts) return fail(ctx, CFBPE_EINVAL, "out_ids and out_starts are required");
    return run_host(ctx, n_prompts, bytes, offsets, vocab_ids, out_ids, out_starts, out_cap, out_offsets, out_counts, true);
}

int cfbpe_encode_batch_char_starts(cfbpe_ctx* ctx, uint32_t n_prompts, const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids,
                                   uint32_t unit, uint32_t* out_ids, uint32_t* out_starts, uint64_t out_cap, uint64_t* out_offsets,
                                   uint32_t* out_counts, uint32_t* out_lens) {
    DeviceGuard restore_device;
    if (!ctx) return CFBPE_EINVAL;
    tl_err.clear();
    if (const char* e = unit_args_error(unit, out_ids, out_starts)) return fail(ctx, CFBPE_EINVAL, e);
    const UnitArgs u{unit == CFBPE_UNIT_UTF16 ? 1u : 0u, out_lens};
    return run_host(ctx, n_prompts, bytes, offsets, vocab_ids, out_ids, out_starts, out_cap, out_offsets, out_counts, true, nullptr, nullptr, &u);
}

int cfbpe_count_batch(cfbpe_ctx* ctx, uint32_t n_prompts, const uint8_t* bytes, const uint64_t* offsets,
                      const uint8_t* vocab_ids, uint32_t* out_counts) {
    DeviceGuard restore_device;
    if (!ctx) return CFBPE_EINVAL;
    if (!out_counts && n_prompts) return fail(ctx, CFBPE_EINVAL, "out_counts is NULL");
    return run_host(ctx, n_prompts, bytes, offsets, vocab_ids, nullptr, nullptr, 0, nullptr, out_counts, false);
}

int cfbpe_truncate_batch(cfbpe_ctx* ctx, uint32_t n_prompts, const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids,
                         const uint32_t* budgets, uint32_t mode, uint32_t* out_cut, uint32_t* out_kept, uint32_t* out_counts) {
    DeviceGuard restore_device;
    if (!ctx) return CFBPE_EINVAL;
    tl_err.clear();
    if (const char* e = truncate_args_error(budgets, mode, out_cut, out_kept)) return fail(ctx, CFBPE_EINVAL, e);
    const TruncateArgs t{budgets, mode == CFBPE_TRUNCATE_TAIL ? 1u : 0u, out_cut, out_kept};
    return run_host(ctx, n_prompts, bytes, offsets, vocab_ids, nullptr, nullptr, UINT64_MAX, nullptr, out_counts, true, &t);
}

int cfbpe_chunk_batch(cfbpe_ctx* ctx, uint32_t n_prompts, const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids,
                      uint32_t chunk_tokens, uint32_t overlap_tokens, uint32_t* out_spans, uint64_t chunk_cap, uint64_t* out_chunk_offsets,
                      uint32_t* out_counts) {
    DeviceGuard restore_device;
    if (!ctx) return CFBPE_EINVAL;
    tl_err.clear();
    if (const char* e = chunk_args_error(chunk_tokens, overlap_tokens, out_spans, out_chunk_offsets)) return fail(ctx, CFBPE_EINVAL, e);
    const ChunkArgs c{chunk_tokens, chunk_tokens - overlap_tokens, out_spans, chunk_cap, out_chunk_offsets, nullptr};
    return run_host(ctx, n_prompts, bytes, offsets, vocab_ids, nullptr, nullptr, UINT64_MAX, nullptr, out_counts, true, nullptr, &c);
}

int cfbpe_decode_batch(cfbpe_ctx* ctx, uint32_t n_seqs, const uint32_t* ids, const uint64_t* id_offsets,
                       const uint8_t* vocab_ids, uint8_t* out_bytes, uint64_t out_cap, uint64_t* out_offsets) {
    DeviceGuard restore_device;
    if (!ctx) return CFBPE_EINVAL;
    tl_err.clear();
    std::shared_lock<std::shared_mutex> vocabs(ctx->vocab_mu);
    if (!id_offsets || !out_offsets) return fail(ctx, CFBPE_EINVAL, "offsets pointer is NULL");
    if (n_seqs > ctx->max_prompts) return fail(ctx, CFBPE_EINVAL, "batch exceeds the limits of this context");
    if (id_offsets[0] != 0) return fail(ctx, CFBPE_EINVAL, "id_offsets[0] must be 0");
    for (uint32_t i = 0; i < n_seqs; ++i) if (id_offsets[i + 1] < id_offsets[i]) return fail(ctx, CFBPE_EINVAL, "id_offsets must not decrease");
    const uint64_t n_ids = id_offsets[n_seqs];
    if (n_ids > ctx->max_bytes) return fail(ctx, CFBPE_EINVAL, "batch exceeds the limits of this context");
    if (n_ids && !ids) return fail(ctx, CFBPE_EINVAL, "ids is NULL");
    for (uint32_t i = 0; vocab_ids && i < n_seqs; ++i)
        if (vocab_ids[i] >= kMaxVocabs || !ctx->vocabs[vocab_ids[i]].loaded) return fail(ctx, CFBPE_ENOENT, "vocab " + std::to_string(vocab_ids[i]) + " is not loaded");
    if (!vocab_ids && !ctx->vocabs[0].loaded) return fail(ctx, CFBPE_ENOENT, "vocab 0 is not loaded");
    DeviceCtx* dv = ctx->devs[0].get();      // (decode runs on the first device: it is not on the hot path)
    LaneLock lk(dv);
    Lane* ln = lk.ln;
    CK(cudaSetDevice(dv->device));
    const int rc = wait_for_device_call(ctx, ln);
    if (rc) return rc;
    cudaStream_t s = ln->stream.get();
    if (n_ids) CK(cudaMemcpyAsync(ln->d_out_ids.get(), ids, n_ids * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(ln->d_offsets.get(), id_offsets, (static_cast<uint64_t>(n_seqs) + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
    if (vocab_ids && n_seqs) CK(cudaMemcpyAsync(ln->d_vocab_ids.get(), vocab_ids, n_seqs, cudaMemcpyHostToDevice, s));
    CK(cudaMemsetAsync(ln->ws.status, 0, sizeof(DeviceStatus), s));
    DecodeView d{ln->d_out_ids.get(), ln->d_offsets.get(), vocab_ids ? ln->d_vocab_ids.get() : nullptr, n_seqs, n_ids};
    const uint32_t n_tiles = static_cast<uint32_t>((n_ids + kDecodeTile - 1) / kDecodeTile);
    if (n_tiles) decode_len_kernel<<<n_tiles, 256, 0, s>>>(d, dv->vs, ln->ws.ids_by_pos, ln->d_dec_sums.get(), ln->ws.status, dv->specials);
    tile_scan_kernel<<<1, n_tiles ? 1024 : 32, 0, s>>>(ln->d_dec_sums.get(), n_tiles, ln->d_dec_base.get(), ln->ws.status, nullptr);
    if (n_tiles) decode_copy_kernel<<<n_tiles, 256, 0, s>>>(d, dv->vs, ln->ws.ids_by_pos, ln->d_dec_base.get(), ln->d_bytes.get(), ctx->max_bytes, dv->specials);
    decode_offsets_kernel<<<static_cast<unsigned>((static_cast<uint64_t>(n_seqs) + 1 + 255) / 256), 256, 0, s>>>(d, ln->ws.ids_by_pos, ln->d_dec_base.get(), ln->d_out_offsets.get(), ln->ws.status);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(ln->h_status.get(), ln->ws.status, sizeof(DeviceStatus), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    const DeviceStatus st = *ln->h_status;
    if (st.bad_utf8) return fail(ctx, CFBPE_EINVAL, "a token id is outside its vocabulary");
    const uint64_t total = st.tok_end;
    if (total > ctx->max_bytes) return fail(ctx, CFBPE_EINVAL, "the decoded batch exceeds max_batch_bytes of this context");
    CK(cudaMemcpyAsync(out_offsets, ln->d_out_offsets.get(), (static_cast<uint64_t>(n_seqs) + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
    if (total > out_cap || (total && !out_bytes)) {
        CK(cudaStreamSynchronize(s));
        out_offsets[n_seqs] = total;
        return fail(ctx, CFBPE_ENOSPC, "out_cap too small: need " + std::to_string(total) + " bytes");
    }
    if (total) CK(cudaMemcpyAsync(out_bytes, ln->d_bytes.get(), total, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return CFBPE_OK;
}

int cfbpe_encode_batch_device(cfbpe_ctx* ctx, uint32_t n_prompts, const uint8_t* d_bytes, uint64_t total_bytes,
                              const uint64_t* d_offsets, const uint8_t* d_vocab_ids, uint32_t* d_out_ids,
                              uint64_t out_cap, uint64_t* d_out_offsets, uint32_t* d_out_counts, uint64_t* n_tokens,
                              void* stream) {
    DeviceGuard restore_device;
    if (!ctx) return CFBPE_EINVAL;
    tl_err.clear();
    return run_device(ctx, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, d_out_ids, nullptr, out_cap, d_out_offsets, d_out_counts,
                      n_tokens, stream);
}

int cfbpe_encode_batch_starts_device(cfbpe_ctx* ctx, uint32_t n_prompts, const uint8_t* d_bytes, uint64_t total_bytes, const uint64_t* d_offsets,
                                     const uint8_t* d_vocab_ids, uint32_t* d_out_ids, uint32_t* d_out_starts, uint64_t out_cap,
                                     uint64_t* d_out_offsets, uint32_t* d_out_counts, uint64_t* n_tokens, void* stream) {
    DeviceGuard restore_device;
    if (!ctx) return CFBPE_EINVAL;
    tl_err.clear();
    if (!d_out_ids || !d_out_starts) return fail(ctx, CFBPE_EINVAL, "d_out_ids and d_out_starts are required");
    return run_device(ctx, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, d_out_ids, d_out_starts, out_cap, d_out_offsets, d_out_counts,
                      n_tokens, stream);
}

int cfbpe_encode_batch_char_starts_device(cfbpe_ctx* ctx, uint32_t n_prompts, const uint8_t* d_bytes, uint64_t total_bytes,
                                          const uint64_t* d_offsets, const uint8_t* d_vocab_ids, uint32_t unit, uint32_t* d_out_ids,
                                          uint32_t* d_out_starts, uint64_t out_cap, uint64_t* d_out_offsets, uint32_t* d_out_counts,
                                          uint32_t* d_out_lens, uint64_t* n_tokens, void* stream) {
    DeviceGuard restore_device;
    if (!ctx) return CFBPE_EINVAL;
    tl_err.clear();
    if (const char* e = unit_args_error(unit, d_out_ids, d_out_starts)) return fail(ctx, CFBPE_EINVAL, e);
    const UnitView uv{unit == CFBPE_UNIT_UTF16 ? 1u : 0u, d_out_lens};
    return run_device(ctx, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, d_out_ids, d_out_starts, out_cap, d_out_offsets, d_out_counts,
                      n_tokens, stream, &uv);
}

int cfbpe_truncate_batch_device(cfbpe_ctx* ctx, uint32_t n_prompts, const uint8_t* d_bytes, uint64_t total_bytes, const uint64_t* d_offsets,
                                const uint8_t* d_vocab_ids, const uint32_t* d_budgets, uint32_t mode, uint32_t* d_out_cut, uint32_t* d_out_kept,
                                uint32_t* d_out_counts, void* stream) {
    DeviceGuard restore_device;
    if (!ctx) return CFBPE_EINVAL;
    tl_err.clear();
    if (const char* e = truncate_args_error(d_budgets, mode, d_out_cut, d_out_kept)) return fail(ctx, CFBPE_EINVAL, e);
    return run_device_truncate(ctx, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, d_budgets, mode, d_out_cut, d_out_kept, d_out_counts,
                               stream);
}

int cfbpe_chunk_batch_device(cfbpe_ctx* ctx, uint32_t n_prompts, const uint8_t* d_bytes, uint64_t total_bytes, const uint64_t* d_offsets,
                             const uint8_t* d_vocab_ids, uint32_t chunk_tokens, uint32_t overlap_tokens, uint32_t* d_out_spans, uint64_t chunk_cap,
                             uint64_t* d_out_chunk_offsets, uint32_t* d_out_counts, uint64_t* n_chunks, void* stream) {
    DeviceGuard restore_device;
    if (!ctx) return CFBPE_EINVAL;
    tl_err.clear();
    if (const char* e = chunk_args_error(chunk_tokens, overlap_tokens, d_out_spans, d_out_chunk_offsets)) return fail(ctx, CFBPE_EINVAL, e);
    return run_device_chunk(ctx, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, chunk_tokens, overlap_tokens, d_out_spans, chunk_cap,
                            d_out_chunk_offsets, d_out_counts, n_chunks, stream);
}

int cfbpe_vocab_set_specials(cfbpe_ctx* ctx, uint32_t vocab_id, uint32_t n, const uint8_t* bytes, const uint64_t* offsets, const uint32_t* ids) {
    DeviceGuard restore_device;
    if (!ctx) return CFBPE_EINVAL;
    tl_err.clear();
    if (vocab_id >= CFBPE_MAX_VOCABS) return fail(ctx, CFBPE_EINVAL, "vocab_id out of range");
    std::vector<uint32_t> words;
    std::string e;
    const int rc = build_special_table(n, bytes, offsets, ids, words, e);
    if (rc) return fail(ctx, rc, e);
    std::unique_lock<std::shared_mutex> lock(ctx->vocab_mu);
    if (!ctx->vocabs[vocab_id].loaded) return fail(ctx, CFBPE_ENOENT, "vocab " + std::to_string(vocab_id) + " is not loaded");
    const size_t G = ctx->devs.size();
    std::vector<DevPtr<uint32_t>> nt(G);      // the new tables, one a device: released on return unless installed
    if (!words.empty()) {
        for (size_t d = 0; d < G; ++d) {      // a plain copy to every device: the table is a few KB
            cudaSetDevice(ctx->devs[d]->device);
            cudaError_t ce = dmalloc(nt[d], words.size());
            if (ce == cudaSuccess) ce = cudaMemcpy(nt[d].get(), words.data(), words.size() * sizeof(uint32_t), cudaMemcpyHostToDevice);
            if (ce != cudaSuccess) {
                cudaGetLastError();
                return fail(ctx, CFBPE_ENOMEM, std::string("special-token table upload: ") + cudaGetErrorString(ce));
            }
        }
    }
    clear_specials(ctx, vocab_id);
    ctx->specials[vocab_id] = std::move(words);
    for (size_t d = 0; d < G; ++d) {
        DeviceCtx* dv = ctx->devs[d].get();
        dv->d_specials[vocab_id] = std::move(nt[d]);
        dv->specials.v[vocab_id] = make_special_view(dv->d_specials[vocab_id].get(), ctx->specials[vocab_id]);
    }
    return CFBPE_OK;
}

int cfbpe_encode_batch_special(cfbpe_ctx* ctx, uint32_t n_prompts, const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids,
                               const uint8_t* const* modes, uint32_t* out_ids, uint64_t out_cap, uint64_t* out_offsets, uint32_t* out_counts,
                               uint32_t* out_bad) {
    DeviceGuard restore_device;
    if (!ctx) return CFBPE_EINVAL;
    return run_host_special(ctx, n_prompts, bytes, offsets, vocab_ids, modes, out_ids, out_cap, out_offsets, out_counts, out_bad);
}

int cfbpe_encode_batch_special_device(cfbpe_ctx* ctx, uint32_t n_prompts, const uint8_t* d_bytes, uint64_t total_bytes, const uint64_t* d_offsets,
                                      const uint8_t* d_vocab_ids, const uint8_t* const* modes, uint32_t* d_out_ids, uint64_t out_cap,
                                      uint64_t* d_out_offsets, uint32_t* d_out_counts, uint64_t* n_tokens, uint32_t* out_bad, void* stream) {
    DeviceGuard restore_device;
    if (!ctx) return CFBPE_EINVAL;
    tl_err.clear();
    return run_device_special(ctx, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, modes, d_out_ids, out_cap, d_out_offsets, d_out_counts,
                              n_tokens, out_bad, stream);
}

int cfbpe_encode_batch_lossy(cfbpe_ctx* ctx, uint32_t n_prompts, const uint8_t* bytes, const uint64_t* offsets, const uint8_t* vocab_ids,
                             uint32_t* out_ids, uint64_t out_cap, uint64_t* out_offsets, uint32_t* out_counts, uint32_t* out_replaced) {
    DeviceGuard restore_device;
    if (!ctx) return CFBPE_EINVAL;
    return run_host_lossy(ctx, n_prompts, bytes, offsets, vocab_ids, out_ids, out_cap, out_offsets, out_counts, out_replaced);
}

int cfbpe_encode_batch_lossy_device(cfbpe_ctx* ctx, uint32_t n_prompts, const uint8_t* d_bytes, uint64_t total_bytes, const uint64_t* d_offsets,
                                    const uint8_t* d_vocab_ids, uint32_t* d_out_ids, uint64_t out_cap, uint64_t* d_out_offsets,
                                    uint32_t* d_out_counts, uint32_t* d_out_replaced, uint64_t* n_tokens, void* stream) {
    DeviceGuard restore_device;
    if (!ctx) return CFBPE_EINVAL;
    tl_err.clear();
    return run_device_lossy(ctx, n_prompts, d_bytes, total_bytes, d_offsets, d_vocab_ids, d_out_ids, out_cap, d_out_offsets, d_out_counts,
                            d_out_replaced, n_tokens, stream);
}

int cfbpe_device_status(cfbpe_ctx* ctx, void* stream) {
    DeviceGuard restore_device;
    if (!ctx) return CFBPE_EINVAL;
    Lane* ln = tl_device_lane;      // the lane of this thread's last device-path call
    if (!ln) return CFBPE_OK;
    std::lock_guard<std::mutex> lock(ln->mu);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    CK(cudaSetDevice(ln->device));
    CK(cudaMemcpyAsync(ln->h_status.get(), ln->ws.status, sizeof(DeviceStatus), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    return device_call_status(ctx, ln);
}

void* cfbpe_host_alloc(cfbpe_ctx* ctx, size_t size) {
    DeviceGuard restore_device;
    if (!ctx) return nullptr;
    void* p = nullptr;
    cudaSetDevice(ctx->devs[0]->device);
    if (cudaMallocHost(&p, size ? size : 1) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
void cfbpe_host_free(cfbpe_ctx* ctx, void* ptr) {
    DeviceGuard restore_device;
    if (!ctx || !ptr) return;
    HostFree{}(ptr);
}

int cfbpe_profile_enable(cfbpe_ctx* ctx, int on) {
    if (!ctx) return CFBPE_EINVAL;
    ctx->profiling.store(on != 0);
    tl_profile_ready = false;
    return CFBPE_OK;
}
int cfbpe_profile_read(cfbpe_ctx* ctx, cfbpe_profile* out) {
    DeviceGuard restore_device;
    if (!ctx || !out) return CFBPE_EINVAL;
    if (!tl_profile_ready) return CFBPE_ENOENT;
    *out = tl_profile;
    return CFBPE_OK;
}

}  // extern "C"
