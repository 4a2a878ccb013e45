// TEST TOOLING ONLY -- host emulation of the tiny slice of the CUDA runtime and
// execution model that the SwiFTly kernels use, so that the kernel *bodies*
// (index algebra, FFT passes, barriers) can be exercised by pytest in a
// container without a GPU.  Each CUDA thread of a CTA runs as a ucontext fibre;
// __syncthreads() yields to a round-robin scheduler, which reproduces barrier
// semantics exactly (one sweep = every thread advances to its next barrier).
// The product library is never built from this header.
#pragma once

#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <ucontext.h>

#include <vector>

struct double2 {
    double x, y;
};
static inline double2 make_double2(double x, double y) {
    double2 r;
    r.x = x;
    r.y = y;
    return r;
}

typedef int cudaError_t;
typedef void* cudaStream_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2, cudaErrorInvalidValue = 1 };
enum cudaMemcpyKind {
    cudaMemcpyHostToHost = 0,
    cudaMemcpyHostToDevice = 1,
    cudaMemcpyDeviceToHost = 2,
    cudaMemcpyDeviceToDevice = 3,
    cudaMemcpyDefault = 4
};

static inline cudaError_t cudaMalloc(void** p, size_t n) {
    *p = malloc(n ? n : 1);
    return *p ? cudaSuccess : cudaErrorMemoryAllocation;
}
static inline cudaError_t cudaFree(void* p) {
    free(p);
    return cudaSuccess;
}
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) {
    memmove(d, s, n);
    return cudaSuccess;
}
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t) {
    memmove(d, s, n);
    return cudaSuccess;
}
static inline cudaError_t cudaMemcpy2DAsync(void* d, size_t dp, const void* s, size_t sp, size_t w,
                                            size_t h, cudaMemcpyKind, cudaStream_t) {
    for (size_t i = 0; i < h; ++i) memmove((char*)d + i * dp, (const char*)s + i * sp, w);
    return cudaSuccess;
}
static inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t) {
    memset(d, v, n);
    return cudaSuccess;
}
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int* d) {
    *d = 0;
    return cudaSuccess;
}
static inline const char* cudaGetErrorString(cudaError_t) { return "emulated CUDA error"; }

namespace swiftly {

struct EmuBlock;

struct HostCtx {
    int tid, bid, nblocks;
    char* smem;
    const void* tmaps;
    EmuBlock* blk;
    inline void sync() const;
    // named barriers with the hardware's counting semantics (bar.sync / bar.arrive a, b):
    // the barrier completes when `count` threads have arrived; bar.sync waits for that,
    // bar.arrive does not.  A protocol error (unbalanced arrivals) shows up as a deadlock,
    // which the scheduler detects and reports instead of hanging; an id above 15 or a count
    // that is not whole warps on a named barrier is reported as soon as it is used.
    inline void group_sync(int id, int count) const;
    inline void group_arrive(int id, int count) const;
    inline void yield() const;
    // bulk asynchronous copies tracked by an mbarrier: the emulated copy completes immediately
    // (races between the asynchronous copy and ordinary accesses are NOT modelled), but the
    // barrier's transaction protocol is accounted for, see EmuTxBarrier below
    inline void tx_init(uint64_t* bar) const;
    inline void tx_expect(uint64_t* bar, uint32_t bytes) const;
    inline void tx_copy(void* dst, const void* src, uint32_t bytes, uint64_t* bar) const;
    inline void tx_wait(uint64_t* bar, uint32_t parity) const;
    inline void bulk_prefetch_l2(const void*, uint32_t) const {}
    inline void nap(unsigned) const {}
    inline void fence_async() const {}
    inline void bulk_commit() const {}
    inline void bulk_wait_read() const {}
    inline void bulk_wait_all() const {}
    inline void tensor_store(const void* map, const void* smem_src, int c1, int c2, int c3) const;
    inline void tensor_load(void* smem_dst, const void* map, int c1, int c2, uint64_t* bar) const;
    // parking space (global scratch on the device): plain host memory
    inline void park_st(double2* p, double2 v) const { *p = v; }
    inline double2 park_ld(const double2* p) const { return *p; }
};

}  // namespace swiftly
namespace swiftly {
struct TensorMap4;
void emu_tensor_store(const TensorMap4* map, const double* src, int c1, int c2, int c3);
void emu_tensor_load(const TensorMap4* map, double* dst, int c1, int c2);
// the bytes a load delivers: the full box, zero fill included
uint32_t emu_tensor_box_bytes(const TensorMap4* map);
inline void HostCtx::tensor_store(const void* map, const void* smem_src, int c1, int c2,
                                  int c3) const {
    emu_tensor_store((const TensorMap4*)map, (const double*)smem_src, c1, c2, c3);
}

// State of one bulk-copy barrier (an mbarrier initialised with count 1, as DeviceCtx::tx_init
// does) of the running CTA.  The hardware completes a phase when the arming thread has arrived
// (tx_expect) and the bytes it announced have been delivered; a wait on parity p returns once the
// phase of that parity is complete.  A protocol slip therefore hangs the CTA or lets it read a
// row that has not landed.  The emulator reports instead:
//   * tx_expect on a barrier whose current phase is already armed;
//   * a copy arriving on a barrier that is not armed, or delivering more bytes than are left;
//   * tx_wait with the wrong parity -- every thread of the CTA waits on every phase once, in
//     order (so do all kernels of the library), hence a thread's k-th wait takes parity k & 1;
//   * tx_wait on a phase that is not complete: the emulated copies are synchronous, so bytes
//     still missing when the wait is reached never arrive;
//   * a phase completing while some thread has not yet waited on the phase before it: that
//     thread's wait would be answered by the wrong phase.
struct EmuTxBarrier {
    uint64_t* bar;
    bool armed;
    uint32_t pending;             // bytes the current phase still expects
    unsigned phases;              // completed phases
    std::vector<unsigned> waits;  // per thread: waits done
};

struct EmuBlock {
    std::vector<EmuTxBarrier> tx;
    ucontext_t main_ctx;
    std::vector<ucontext_t> ctxs;
    std::vector<char*> stacks;
    std::vector<char> done;
    int current;
    void (*entry)(void*, HostCtx&);
    void* body;
    std::vector<HostCtx> hctx;
    int nthreads;
    int bar_arrived[16];
    unsigned bar_gen[16];
    unsigned long progress;  // barrier completions + thread exits (deadlock detection)
};

static EmuBlock* g_emu_block = nullptr;

inline void HostCtx::yield() const {
    EmuBlock* b = blk;
    swapcontext(&b->ctxs[tid], &b->main_ctx);
}

// bar.sync / bar.arrive take ids 0..15, and a thread count that is a multiple of the warp size
// (barrier 0 is __syncthreads, whose count is the whole CTA): anything else is invalid on the
// hardware, so the emulator reports it as a protocol error, like a deadlock.  A CTA of less than
// one warp cannot form a whole-warp barrier at all: it is a kernel form forced at a line length
// far below the one it serves on the GPU (the split K2 forms at yN = 512: 16-thread CTAs, whole
// warps at yN = 16384), and only the id range is checked there.
static inline void emu_check_barrier(int id, int count, int cta_threads) {
    const bool warps = count > 0 && (count % 32 == 0 || cta_threads < 32);
    if (id < 0 || id >= 16 || (id != 0 && !warps)) {
        fprintf(stderr, "swiftly emulator: barrier PROTOCOL error (id %d, count %d): named barriers "
                        "take ids 0..15 and whole warps\n", id, count);
        abort();
    }
}

static inline void emu_tx_error(const HostCtx& c, const char* what, const EmuTxBarrier* b) {
    fprintf(stderr, "swiftly emulator: bulk-copy barrier PROTOCOL error in block %d, thread %d: %s",
            c.bid, c.tid, what);
    if (b)
        fprintf(stderr, " (%u phases complete, current phase %s, %u bytes outstanding)", b->phases,
                b->armed ? "armed" : "not armed", b->pending);
    fprintf(stderr, "\n");
    abort();
}

static inline EmuTxBarrier& emu_tx_find(const HostCtx& c, uint64_t* bar) {
    for (EmuTxBarrier& b : c.blk->tx)
        if (b.bar == bar) return b;
    emu_tx_error(c, "barrier used before tx_init", nullptr);
    abort();
}

static inline void emu_tx_deliver(const HostCtx& c, uint64_t* bar, uint32_t bytes) {
    EmuTxBarrier& b = emu_tx_find(c, bar);
    if (!b.armed) emu_tx_error(c, "copy arrives on a barrier that is not armed", &b);
    if (bytes > b.pending) emu_tx_error(c, "copy delivers more bytes than tx_expect announced", &b);
    b.pending -= bytes;
    if (b.pending) return;
    for (unsigned w : b.waits)
        if (w < b.phases)
            emu_tx_error(c, "phase completes before every thread waited on the previous one", &b);
    b.armed = false;
    ++b.phases;
}

inline void HostCtx::tx_init(uint64_t* bar) const {
    EmuTxBarrier fresh{bar, false, 0, 0, std::vector<unsigned>(blk->nthreads, 0u)};
    for (EmuTxBarrier& b : blk->tx)
        if (b.bar == bar) {
            b = fresh;
            return;
        }
    blk->tx.push_back(fresh);
}

inline void HostCtx::tx_expect(uint64_t* bar, uint32_t bytes) const {
    EmuTxBarrier& b = emu_tx_find(*this, bar);
    if (b.armed) emu_tx_error(*this, "tx_expect on a phase that is already armed", &b);
    b.armed = true;
    b.pending = bytes;
    if (!bytes) emu_tx_deliver(*this, bar, 0);
}

inline void HostCtx::tx_copy(void* dst, const void* src, uint32_t bytes, uint64_t* bar) const {
    memcpy(dst, src, bytes);
    emu_tx_deliver(*this, bar, bytes);
}

inline void HostCtx::tensor_load(void* smem_dst, const void* map, int c1, int c2,
                                 uint64_t* bar) const {
    emu_tensor_load((const TensorMap4*)map, (double*)smem_dst, c1, c2);
    emu_tx_deliver(*this, bar, emu_tensor_box_bytes((const TensorMap4*)map));
}

inline void HostCtx::tx_wait(uint64_t* bar, uint32_t parity) const {
    EmuTxBarrier& b = emu_tx_find(*this, bar);
    const unsigned k = b.waits[tid];
    if ((k & 1u) != (parity & 1u))
        emu_tx_error(*this, "tx_wait with the parity of the wrong phase", &b);
    if (b.phases <= k) emu_tx_error(*this, "tx_wait on a phase that cannot complete", &b);
    b.waits[tid] = k + 1;
}

inline void HostCtx::group_arrive(int id, int count) const {
    EmuBlock* b = blk;
    emu_check_barrier(id, count, b->nthreads);
    if (++b->bar_arrived[id] >= count) {
        b->bar_arrived[id] = 0;
        ++b->bar_gen[id];
        ++b->progress;
    }
}

inline void HostCtx::group_sync(int id, int count) const {
    EmuBlock* b = blk;
    const unsigned g = b->bar_gen[id];
    group_arrive(id, count);
    while (b->bar_gen[id] == g) yield();
}

inline void HostCtx::sync() const { group_sync(0, blk->nthreads); }

static void emu_trampoline() {
    EmuBlock* b = g_emu_block;
    int t = b->current;
    b->entry(b->body, b->hctx[t]);
    b->done[t] = 1;
    ++b->progress;
    // returning switches to uc_link (main_ctx)
}

template <class Body>
static void emu_entry(void* body, HostCtx& ctx) {
    (*(const Body*)body)(ctx);
}

template <class Body>
inline cudaError_t launch_body_impl(const Body& body, const void* tmaps, int grid, size_t smem_bytes);

template <class Body>
inline cudaError_t launch_body(const Body& body, int grid, size_t smem_bytes, cudaStream_t) {
    return launch_body_impl(body, nullptr, grid, smem_bytes);
}

template <class Body>
inline cudaError_t launch_body_maps(const Body& body, const typename Body::Maps& maps, int grid,
                                    size_t smem_bytes, cudaStream_t) {
    return launch_body_impl(body, &maps, grid, smem_bytes);
}

template <class Body>
inline cudaError_t launch_body_impl(const Body& body, const void* tmaps, int grid, size_t smem_bytes) {
    const int T = Body::THREADS;
    const size_t STACK = 256 * 1024;
    EmuBlock blk;
    blk.ctxs.resize(T);
    blk.stacks.resize(T);
    blk.done.resize(T);
    blk.hctx.resize(T);
    blk.entry = &emu_entry<Body>;
    blk.body = (void*)&body;
    for (int t = 0; t < T; ++t) blk.stacks[t] = (char*)malloc(STACK);
    char* smem = (char*)malloc(smem_bytes + 64);
    for (int bid = 0; bid < grid; ++bid) {
        memset(smem, 0xA5, smem_bytes + 64);  // poison: uninitialised smem reads show up
        for (int t = 0; t < T; ++t) {
            getcontext(&blk.ctxs[t]);
            blk.ctxs[t].uc_stack.ss_sp = blk.stacks[t];
            blk.ctxs[t].uc_stack.ss_size = STACK;
            blk.ctxs[t].uc_link = &blk.main_ctx;
            makecontext(&blk.ctxs[t], (void (*)())emu_trampoline, 0);
            blk.done[t] = 0;
            blk.hctx[t].tid = t;
            blk.hctx[t].bid = bid;
            blk.hctx[t].nblocks = grid;
            blk.hctx[t].smem = smem;
            blk.hctx[t].tmaps = tmaps;
            blk.hctx[t].blk = &blk;
        }
        g_emu_block = &blk;
        blk.nthreads = T;
        blk.tx.clear();
        for (int i = 0; i < 16; ++i) {
            blk.bar_arrived[i] = 0;
            blk.bar_gen[i] = 0;
        }
        blk.progress = 0;
        bool any = true;
        int idle_sweeps = 0;
        while (any) {
            any = false;
            const unsigned long before = blk.progress;
            for (int t = 0; t < T; ++t) {
                if (blk.done[t]) continue;
                blk.current = t;
                swapcontext(&blk.main_ctx, &blk.ctxs[t]);
                if (!blk.done[t]) any = true;
            }
            // a sweep lets every live thread run to its next wait; two sweeps in a row without
            // a barrier completing or a thread finishing means nobody can ever proceed
            idle_sweeps = (any && blk.progress == before) ? idle_sweeps + 1 : 0;
            if (idle_sweeps >= 2) {
                fprintf(stderr, "swiftly emulator: barrier DEADLOCK in block %d (arrivals:", bid);
                for (int i = 0; i < 16; ++i) fprintf(stderr, " %d", blk.bar_arrived[i]);
                fprintf(stderr, ")\n");
                abort();
            }
        }
    }
    free(smem);
    for (int t = 0; t < T; ++t) free(blk.stacks[t]);
    return cudaSuccess;
}

}  // namespace swiftly
