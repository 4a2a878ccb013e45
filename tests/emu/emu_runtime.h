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
    // bulk asynchronous copies: the emulated copy completes immediately (races between the
    // asynchronous copy and ordinary accesses are NOT modelled -- only the index algebra is)
    inline void tx_init(uint64_t* bar) const { *bar = 0; }
    inline void tx_expect(uint64_t*, uint32_t) const {}
    inline void tx_copy(void* dst, const void* src, uint32_t bytes, uint64_t* bar) const {
        memcpy(dst, src, bytes);
        *bar += 1;
    }
    inline void tx_wait(uint64_t*, uint32_t) const {}
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
inline void HostCtx::tensor_load(void* smem_dst, const void* map, int c1, int c2,
                                 uint64_t* bar) const {
    emu_tensor_load((const TensorMap4*)map, (double*)smem_dst, c1, c2);
    *bar += 1;
}
inline void HostCtx::tensor_store(const void* map, const void* smem_src, int c1, int c2,
                                  int c3) const {
    emu_tensor_store((const TensorMap4*)map, (const double*)smem_src, c1, c2, c3);
}

struct EmuBlock {
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
