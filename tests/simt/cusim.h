// cusim.h -- a small CPU SIMT emulator for running the product's CUDA kernels WITHOUT a GPU.
//
// TEST INFRASTRUCTURE.  The build container has no GPU and every GPU call is minutes of queue
// time, so the non-GPU test suite compiles cyberfabric-core_b200/csrc/bpe_kernels.cuh
// (unchanged) as plain C++ against this header and runs the kernels here: every CUDA thread is
// a fiber (hand-rolled x86-64 context switch), warp collectives (__shfl_*_sync, __ballot_sync,
// ...) and __syncthreads() are rendezvous points between fibers, atomics are plain operations
// (one OS thread runs one block at a time).  A collective that not all live lanes of a warp
// reach is reported as a deadlock instead of hanging -- the same bug would be UB on the GPU.
//
// This is not a CPU fallback: libcfbpe.so contains none of it and fails without a device.
#pragma once
#define CUSIM_EMULATOR 1
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>

namespace cusim {

struct uint3_t { unsigned x, y, z; };

struct Fiber {
    void* sp = nullptr;
    char* stack = nullptr;
    uint3_t tid{0, 0, 0};
    bool done = false;
};

struct WarpState {
    uint32_t arrived = 0;
    uint64_t gen = 0;
    uint64_t vals[2][32];
    uint32_t exited = 0;
};

struct BlockState {
    std::vector<Fiber> fibers;
    std::vector<WarpState> warps;
    unsigned nthreads = 0;
    unsigned n_done = 0;
    unsigned bar_arrived = 0;
    uint64_t bar_gen = 0;
    uint64_t progress = 0;  // bumped on every completed rendezvous / exit
    uint3_t bid{0, 0, 0}, bdim{1, 1, 1}, gdim{1, 1, 1};
    std::function<void()> body;
    void* sched_sp = nullptr;
    Fiber* cur = nullptr;
};

inline BlockState& B() { static BlockState b; return b; }

extern "C" void cusim_switch(void** from_sp, void* to_sp);
asm(R"(
.text
.globl cusim_switch
.type cusim_switch,@function
cusim_switch:
    pushq %rbp
    pushq %rbx
    pushq %r12
    pushq %r13
    pushq %r14
    pushq %r15
    movq %rsp, (%rdi)
    movq %rsi, %rsp
    popq %r15
    popq %r14
    popq %r13
    popq %r12
    popq %rbx
    popq %rbp
    ret
.size cusim_switch,.-cusim_switch
)");

inline void yield() {
    BlockState& b = B();
    cusim_switch(&b.cur->sp, b.sched_sp);
}

inline void fiber_main() {
    BlockState& b = B();
    b.body();
    Fiber* f = b.cur;
    f->done = true;
    b.n_done++;
    b.progress++;
    b.warps[f->tid.x >> 5].exited |= 1u << (f->tid.x & 31);
    // an exit may complete a rendezvous the rest of the warp is waiting in
    WarpState& w = b.warps[f->tid.x >> 5];
    unsigned lanes = b.nthreads - (f->tid.x & ~31u);
    uint32_t exist = lanes >= 32 ? 0xFFFFFFFFu : ((1u << lanes) - 1u);
    if (w.arrived && w.arrived == (exist & ~w.exited)) { w.arrived = 0; w.gen++; }
    if (b.bar_arrived && b.bar_arrived == b.nthreads - b.n_done) { b.bar_arrived = 0; b.bar_gen++; }
    yield();
    std::fprintf(stderr, "cusim: resumed a finished fiber\n");
    std::abort();
}

constexpr size_t kStackBytes = 256 * 1024;

inline void prepare_fiber(Fiber& f) {
    if (!f.stack) f.stack = static_cast<char*>(std::malloc(kStackBytes));
    uintptr_t top = (reinterpret_cast<uintptr_t>(f.stack) + kStackBytes) & ~uintptr_t(15);
    void** sp = reinterpret_cast<void**>(top);
    *--sp = nullptr;                                  // alignment pad
    *--sp = reinterpret_cast<void*>(&fiber_main);     // return address of the first switch
    for (int i = 0; i < 6; ++i) *--sp = nullptr;      // rbp rbx r12 r13 r14 r15
    f.sp = sp;
    f.done = false;
}

inline void run_block() {
    BlockState& b = B();
    b.n_done = 0; b.bar_arrived = 0; b.bar_gen = 0;
    if (b.fibers.size() < b.nthreads) b.fibers.resize(b.nthreads);
    b.warps.assign((b.nthreads + 31) / 32, WarpState());
    for (unsigned t = 0; t < b.nthreads; ++t) { b.fibers[t].tid = {t, 0, 0}; prepare_fiber(b.fibers[t]); }
    while (b.n_done < b.nthreads) {
        const uint64_t before = b.progress;
        for (unsigned t = 0; t < b.nthreads; ++t) {
            Fiber& f = b.fibers[t];
            if (f.done) continue;
            b.cur = &f;
            cusim_switch(&b.sched_sp, f.sp);
        }
        if (b.progress == before) {
            std::fprintf(stderr, "cusim: DEADLOCK in block %u: a collective or __syncthreads() was not reached by all live threads\n", b.bid.x);
            std::abort();
        }
    }
}

template <typename F>
inline void launch(unsigned grid, unsigned block, F&& body) {
    BlockState& b = B();
    b.gdim = {grid, 1, 1};
    b.bdim = {block, 1, 1};
    b.nthreads = block;
    b.body = std::forward<F>(body);
    for (unsigned g = 0; g < grid; ++g) { b.bid = {g, 0, 0}; run_block(); }
}

// ---- rendezvous of the live lanes of the calling fiber's warp; returns the exchange buffer
inline const uint64_t* warp_exchange(uint64_t v) {
    BlockState& b = B();
    const unsigned tid = b.cur->tid.x, lane = tid & 31;
    WarpState& w = b.warps[tid >> 5];
    const uint64_t gen = w.gen;
    uint64_t* buf = w.vals[gen & 1];
    buf[lane] = v;
    w.arrived |= 1u << lane;
    unsigned lanes = b.nthreads - (tid & ~31u);
    uint32_t exist = lanes >= 32 ? 0xFFFFFFFFu : ((1u << lanes) - 1u);
    if (w.arrived == (exist & ~w.exited)) { w.arrived = 0; w.gen++; b.progress++; }
    else while (w.gen == gen) yield();
    return buf;
}
inline uint32_t live_mask() {
    BlockState& b = B();
    const unsigned tid = b.cur->tid.x;
    unsigned lanes = b.nthreads - (tid & ~31u);
    uint32_t exist = lanes >= 32 ? 0xFFFFFFFFu : ((1u << lanes) - 1u);
    return exist & ~b.warps[tid >> 5].exited;
}
inline void syncthreads() {
    BlockState& b = B();
    const uint64_t gen = b.bar_gen;
    b.bar_arrived++;
    if (b.bar_arrived == b.nthreads - b.n_done) { b.bar_arrived = 0; b.bar_gen++; b.progress++; }
    else while (b.bar_gen == gen) yield();
}

inline unsigned char* dyn_smem() { static unsigned char buf[256 * 1024] __attribute__((aligned(16))); return buf; }

template <typename T> inline uint64_t to_u64(T v) { uint64_t u = 0; std::memcpy(&u, &v, sizeof(T)); return u; }
template <typename T> inline T from_u64(uint64_t u) { T v; std::memcpy(&v, &u, sizeof(T)); return v; }

}  // namespace cusim

// ---------------------------------------------------------------------------------------
// CUDA surface
// ---------------------------------------------------------------------------------------
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __launch_bounds__(...)
#define __shared__ static
#define __align__(n) __attribute__((aligned(n)))
// CUDA's alignment: a vector load from a misaligned address faults on the GPU; here the sanitizer build stops on it
struct alignas(16) uint4 { unsigned x, y, z, w; };
struct alignas(8) uint2 { unsigned x, y; };
inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { uint4 v; v.x = x; v.y = y; v.z = z; v.w = w; return v; }
#define threadIdx (cusim::B().cur->tid)
#define blockIdx (cusim::B().bid)
#define blockDim (cusim::B().bdim)
#define gridDim (cusim::B().gdim)

inline void __syncthreads() { cusim::syncthreads(); }
inline void __syncwarp(unsigned = 0xFFFFFFFFu) { cusim::warp_exchange(0); }

template <typename T> inline T __shfl_sync(unsigned, T v, int src) {
    const unsigned lane = threadIdx.x & 31;
    const uint32_t live = cusim::live_mask();
    const uint64_t* buf = cusim::warp_exchange(cusim::to_u64(v));
    const unsigned s = static_cast<unsigned>(src) & 31;
    (void)lane;
    return ((live >> s) & 1u) ? cusim::from_u64<T>(buf[s]) : v;
}
template <typename T> inline T __shfl_down_sync(unsigned, T v, unsigned d) {
    const unsigned lane = threadIdx.x & 31;
    const uint32_t live = cusim::live_mask();
    const uint64_t* buf = cusim::warp_exchange(cusim::to_u64(v));
    const unsigned s = lane + d;
    return (s < 32 && ((live >> s) & 1u)) ? cusim::from_u64<T>(buf[s]) : v;
}
template <typename T> inline T __shfl_up_sync(unsigned, T v, unsigned d) {
    const unsigned lane = threadIdx.x & 31;
    const uint64_t* buf = cusim::warp_exchange(cusim::to_u64(v));
    return (lane >= d) ? cusim::from_u64<T>(buf[lane - d]) : v;
}
template <typename T> inline T __shfl_xor_sync(unsigned, T v, unsigned m) {
    const unsigned lane = threadIdx.x & 31;
    const uint32_t live = cusim::live_mask();
    const uint64_t* buf = cusim::warp_exchange(cusim::to_u64(v));
    const unsigned s = lane ^ m;
    return (s < 32 && ((live >> s) & 1u)) ? cusim::from_u64<T>(buf[s]) : v;
}
inline unsigned __ballot_sync(unsigned, bool pred) {
    const uint32_t live = cusim::live_mask();
    const uint64_t* buf = cusim::warp_exchange(pred ? 1u : 0u);
    unsigned r = 0;
    for (unsigned i = 0; i < 32; ++i) if (((live >> i) & 1u) && buf[i]) r |= 1u << i;
    return r;
}
inline unsigned __reduce_min_sync(unsigned mask, unsigned v) {   // redux.sync.min: min over the lanes named in MY mask
    const uint64_t* buf = cusim::warp_exchange(v);
    unsigned r = 0xFFFFFFFFu;
    for (unsigned i = 0; i < 32; ++i) if ((mask >> i) & 1u) { const unsigned o = static_cast<unsigned>(buf[i]); r = o < r ? o : r; }
    return r;
}
inline unsigned __reduce_or_sync(unsigned mask, unsigned v) {
    const uint64_t* buf = cusim::warp_exchange(v);
    unsigned r = 0;
    for (unsigned i = 0; i < 32; ++i) if ((mask >> i) & 1u) r |= static_cast<unsigned>(buf[i]);
    return r;
}
inline unsigned __reduce_add_sync(unsigned mask, unsigned v) {
    const uint64_t* buf = cusim::warp_exchange(v);
    unsigned r = 0;
    for (unsigned i = 0; i < 32; ++i) if ((mask >> i) & 1u) r += static_cast<unsigned>(buf[i]);
    return r;
}
inline bool __any_sync(unsigned m, bool pred) { return __ballot_sync(m, pred) != 0; }
inline bool __all_sync(unsigned m, bool pred) { return __ballot_sync(m, !pred) == 0; }

inline void __threadfence_system() {}
inline void __threadfence() {}
inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned sh) { sh &= 31; return sh ? ((lo >> sh) | (hi << (32 - sh))) : lo; }
inline int __popc(unsigned x) { return __builtin_popcount(x); }
inline int __popcll(unsigned long long x) { return __builtin_popcountll(x); }
inline int __clz(unsigned x) { return x ? __builtin_clz(x) : 32; }
inline int __clzll(long long x) { return x ? __builtin_clzll(static_cast<unsigned long long>(x)) : 64; }
inline int __ffs(unsigned x) { return __builtin_ffs(static_cast<int>(x)); }
inline int __ffsll(long long x) { return __builtin_ffsll(x); }

template <typename T> inline T atomicOr(T* p, T v) { T o = *p; *p = o | v; return o; }
template <typename T> inline T atomicAdd(T* p, T v) { T o = *p; *p = o + v; return o; }
template <typename T> inline T atomicMin(T* p, T v) { T o = *p; if (v < o) *p = v; return o; }
template <typename T> inline T atomicMax(T* p, T v) { T o = *p; if (v > o) *p = v; return o; }
template <typename T> inline T __ldg(const T* p) { return *p; }
