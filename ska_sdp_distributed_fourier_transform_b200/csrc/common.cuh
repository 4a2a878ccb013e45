// SwiFTly -- common definitions shared by all kernels.
//
// Every kernel body in this library is written as a functor templated on an
// execution context ("Ctx") that provides the thread id, block id, shared
// memory and the CTA barrier.  The CUDA build instantiates the bodies with
// DeviceCtx inside a __global__ entry point.  A second, test-only build
// (tests/emu, -DSWIFTLY_EMU, plain g++) instantiates the very same bodies with
// a host context that runs every CUDA thread as a fibre, so that the index
// algebra of the kernels can be exercised in a container without a GPU.  The
// emulator is test tooling: the product never loads it.
#pragma once

#include <stdint.h>
#include <type_traits>

#if defined(SWIFTLY_EMU)
#include "emu_runtime.h"
#include "emu_cluster.h"
#else
#include <cuda.h>
#include <cuda_runtime.h>
#endif

#if defined(__CUDACC__)
#define SW_HD __host__ __device__ __forceinline__
#define SW_D __device__ __forceinline__
#else
#define SW_HD inline
#define SW_D inline
#endif

namespace swiftly {

typedef double2 cplx;

SW_HD cplx mk(double x, double y) {
    cplx r;
    r.x = x;
    r.y = y;
    return r;
}
SW_HD cplx cadd(cplx a, cplx b) { return mk(a.x + b.x, a.y + b.y); }
SW_HD cplx csub(cplx a, cplx b) { return mk(a.x - b.x, a.y - b.y); }
SW_HD cplx cmul(cplx a, cplx b) { return mk(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
SW_HD cplx cscale(cplx a, double s) { return mk(a.x * s, a.y * s); }
SW_HD cplx cconj(cplx a) { return mk(a.x, -a.y); }
// a * b rounded on its own: never contracted with a following add into one fused multiply-add
SW_HD double mul_rn(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
// multiply by DIR * i   (DIR = -1: forward transform, +1: inverse transform)
template <int DIR>
SW_HD cplx mul_i(cplx a) {
    return DIR < 0 ? mk(a.y, -a.x) : mk(-a.y, a.x);
}

// read-only global load (LDG.E.128 through the non-coherent path on device)
SW_HD cplx ldg_c(const cplx* p) {
#if defined(__CUDA_ARCH__)
    return __ldg(p);
#else
    return *p;
#endif
}
SW_HD double ldg_d(const double* p) {
#if defined(__CUDA_ARCH__)
    return __ldg(p);
#else
    return *p;
#endif
}

// streaming global accesses: data that is touched once per kernel (inputs and outputs are
// far larger than the 50 MB L2) should not push the few reused lines (twiddle / window
// tables, split-kernel scratch) out of L2
SW_HD cplx ld_stream(const cplx* p) {
#if defined(__CUDA_ARCH__)
    return __ldcs(p);
#else
    return *p;
#endif
}
SW_HD double ld_stream_d(const double* p) {
#if defined(__CUDA_ARCH__)
    return __ldcs(p);
#else
    return *p;
#endif
}
SW_HD void st_stream(cplx* p, cplx v) {
#if defined(__CUDA_ARCH__)
    __stcs(p, v);
#else
    *p = v;
#endif
}
SW_HD void st_stream_d(double* p, double v) {
#if defined(__CUDA_ARCH__)
    __stcs(p, v);
#else
    *p = v;
#endif
}

// two adjacent samples (32 bytes, 32-byte aligned): one 32-byte sector per thread, written by
// two streaming 16-byte stores (sm_90 has no 256-bit global store)
SW_HD void st_stream_pair(cplx* p, cplx a, cplx b) {
#if defined(__CUDA_ARCH__)
    __stcs(p, a);
    __stcs(p + 1, b);
#else
    p[0] = a;
    p[1] = b;
#endif
}

// software prefetch of the 32-byte sector(s) holding *p into L2 (no register is tied up):
// all warps of a CTA are in the same phase of a transform, so a plain load at the start of
// the next phase exposes the full DRAM latency; the prefetch is issued one phase ahead
SW_HD void prefetch_l2(const void* p) {
#if defined(__CUDA_ARCH__)
    asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
#else
    (void)p;
#endif
}

// non-negative modulo for possibly negative a, n > 0
SW_HD int64_t pmod(int64_t a, int64_t n) {
    int64_t r = a % n;
    return r < 0 ? r + n : r;
}

// Descriptor of a strided global tile for the TMA engine: rank 4, dimension 0 = (re, im) of a
// complex128 sample, dimensions 1..3 = line / sample / group of an output array in ascending
// stride order.  On the device this is the driver's opaque CUtensorMap (made by
// cuTensorMapEncodeTiled, capi_util.h); the host-emulated test build keeps the plain numbers.
#if defined(SWIFTLY_EMU)
struct TensorMap4 {
    double* base;
    int64_t stride[4];  // in doubles
    int64_t dim[4];
    int box[4];
    int swizzle128;  // loads: destination tile written with the 128-byte swizzle pattern
};
#else
struct alignas(64) TensorMap4 {
    CUtensorMap map;
};
#endif

#if defined(__CUDACC__) && !defined(SWIFTLY_EMU)
// Execution context on the device: one CTA.
struct DeviceCtx {
    int tid, bid, nblocks;
    char* smem;
    const void* tmaps;  // the kernel's tensor maps (a __grid_constant__ parameter) or null
    __device__ __forceinline__ void sync() const { __syncthreads(); }
    // named barrier over `count` threads (a multiple of 32; whole warps), id 1..15
    __device__ __forceinline__ void group_sync(int id, int count) const {
        asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
    }
    // non-blocking arrival at a named barrier (producer side of a bar.sync / bar.arrive pair)
    __device__ __forceinline__ void group_arrive(int id, int count) const {
        asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory");
    }
    // let the calling thread sleep for about `ns` nanoseconds
    __device__ __forceinline__ void nap(unsigned ns) const { __nanosleep(ns); }
    // ---- bulk asynchronous copies (TMA engine, cp.async.bulk) tracked by an mbarrier ----
    // `bar` is an 8-byte shared-memory word; one thread initialises it (count 1 = the thread
    // that issues the copies), everybody waits on its phase parity.
    __device__ __forceinline__ void tx_init(uint64_t* bar) const {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(
                         (uint32_t)__cvta_generic_to_shared(bar)) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    // announce `bytes` of bulk copies for the current phase (issuing thread only)
    __device__ __forceinline__ void tx_expect(uint64_t* bar, uint32_t bytes) const {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(
                         (uint32_t)__cvta_generic_to_shared(bar)), "r"(bytes) : "memory");
    }
    // global -> shared bulk copy (16-byte aligned, size a multiple of 16) completing on `bar`
    __device__ __forceinline__ void tx_copy(void* smem_dst, const void* gmem_src, uint32_t bytes,
                                            uint64_t* bar) const {
        asm volatile(
            "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
            ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gmem_src), "r"(bytes),
              "r"((uint32_t)__cvta_generic_to_shared(bar)) : "memory");
    }
    __device__ __forceinline__ void tx_wait(uint64_t* bar, uint32_t parity) const {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "WAIT_%=:\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
            "@p bra DONE_%=;\n"
            "bra WAIT_%=;\n"
            "DONE_%=:\n"
            "}\n" ::"r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(parity) : "memory");
    }
    // ---- bulk tensor loads (TMA): strided global tile -> shared memory tile, completion on
    // an mbarrier.  Box at coordinates (0, c1, c2, 0) of a rank-4 map; with a 128-byte swizzled
    // map the 16-byte unit u of 128-byte row c of the tile lands at unit (u ^ (c & 7)): strided
    // reads of the tile (every 2nd / 4th sample) are then free of bank conflicts.  The
    // destination must be 1024-byte aligned.
    __device__ __forceinline__ void tensor_load(void* smem_dst, const void* map, int c1, int c2,
                                                uint64_t* bar) const {
        asm volatile(
            "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes "
            "[%0], [%1, {%2, %3, %4, %5}], [%6];"
            ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(map), "r"(0), "r"(c1),
              "r"(c2), "r"(0), "r"((uint32_t)__cvta_generic_to_shared(bar)) : "memory");
    }
    // ---- bulk tensor stores (TMA): shared memory tile -> strided global tile ----
    // ordinary shared-memory writes become visible to the asynchronous proxy
    __device__ __forceinline__ void fence_async() const {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    // store the box at coordinates (0, c1, c2, c3) of a rank-4 tensor map (dimension 0 = the
    // two doubles of a complex sample) from a dense shared-memory tile
    __device__ __forceinline__ void tensor_store(const void* map, const void* smem_src, int c1,
                                                 int c2, int c3) const {
        asm volatile(
            "cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%1, %2, %3, %4}], [%5];"
            ::"l"(map), "r"(0), "r"(c1), "r"(c2), "r"(c3),
              "r"((uint32_t)__cvta_generic_to_shared(smem_src)) : "memory");
    }
    __device__ __forceinline__ void bulk_commit() const {
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    // the bulk stores this thread committed have finished READING shared memory
    __device__ __forceinline__ void bulk_wait_read() const {
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    }
    // ... have completed entirely (their global writes are performed)
    __device__ __forceinline__ void bulk_wait_all() const {
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    }
    // bulk L2 prefetch of a contiguous global region (no registers, no LSU wavefronts)
    __device__ __forceinline__ void bulk_prefetch_l2(const void* gmem_src, uint32_t bytes) const {
        asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gmem_src), "r"(bytes)
                     : "memory");
    }
    // ---- parking space: a per-CTA region of global scratch that stays in the 50 MB L2 ----
    // A thread parks a sample it needs again later in the same CTA (park_st) and takes it back,
    // or -- after a CTA or named barrier -- another thread of the CTA takes it (park_ld).  The
    // accesses bypass L1 (.cg): the parked samples are written and read once per line, and the
    // line's staged row and exchange buffers keep the SM's shared memory.  Kernels lay the
    // region out so that the 32 threads of a warp touch 512 contiguous bytes.
    __device__ __forceinline__ void park_st(cplx* p, cplx v) const { __stcg(p, v); }
    __device__ __forceinline__ cplx park_ld(const cplx* p) const { return __ldcg(p); }
    // ---- thread block clusters (kernels launched with a cluster dimension) ----
    // rank of this CTA in its cluster
    __device__ __forceinline__ int cluster_rank() const {
        uint32_t r;
        asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
        return (int)r;
    }
    // barrier over every thread of the cluster; orders shared-memory accesses across its CTAs
    __device__ __forceinline__ void cluster_sync() const {
        asm volatile("barrier.cluster.arrive.release.aligned;\n"
                     "barrier.cluster.wait.acquire.aligned;" ::: "memory");
    }
    // the shared-memory word of CTA `rank` of the cluster at the offset of the local `p`
    __device__ __forceinline__ static uint32_t peer_addr(const void* p, int rank) {
        uint32_t a;
        asm volatile("mapa.shared::cluster.u32 %0, %1, %2;"
                     : "=r"(a) : "r"((uint32_t)__cvta_generic_to_shared(p)), "r"(rank));
        return a;
    }
    // store into the shared memory of CTA `rank` (distributed shared memory)
    __device__ __forceinline__ void peer_st(cplx* p, int rank, cplx v) const {
        asm volatile("st.shared::cluster.v2.f64 [%0], {%1, %2};"
                     ::"r"(peer_addr(p, rank)), "d"(v.x), "d"(v.y) : "memory");
    }
    // atomic add to a counter in the shared memory of CTA `rank`; returns the previous value
    __device__ __forceinline__ int peer_atomic_add(int* p, int rank, int v) const {
        int prev;
        asm volatile("atom.relaxed.cluster.shared::cluster.add.u32 %0, [%1], %2;"
                     : "=r"(prev) : "r"(peer_addr(p, rank)), "r"(v) : "memory");
        return prev;
    }
    // tx_expect on the bulk-copy barrier of CTA `rank` at the offset of the local `bar`
    __device__ __forceinline__ void tx_expect_peer(uint64_t* bar, int rank, uint32_t bytes) const {
        asm volatile("mbarrier.arrive.expect_tx.shared::cluster.b64 _, [%0], %1;"
                     ::"r"(peer_addr(bar, rank)), "r"(bytes) : "memory");
    }
    // tensor_load / tx_copy delivered to the same offsets in every CTA of `mask`: the data to
    // `smem_dst`, the completion to the barrier at `bar` of each of them
    __device__ __forceinline__ void tensor_load_mc(void* smem_dst, const void* map, int c1, int c2,
                                                   uint64_t* bar, uint16_t mask) const {
        asm volatile(
            "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes"
            ".multicast::cluster [%0], [%1, {%2, %3, %4, %5}], [%6], %7;"
            ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(map), "r"(0), "r"(c1),
              "r"(c2), "r"(0), "r"((uint32_t)__cvta_generic_to_shared(bar)), "h"(mask)
            : "memory");
    }
    __device__ __forceinline__ void tx_copy_mc(void* smem_dst, const void* gmem_src, uint32_t bytes,
                                               uint64_t* bar, uint16_t mask) const {
        asm volatile(
            "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
            " [%0], [%1], %2, [%3], %4;"
            ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gmem_src), "r"(bytes),
              "r"((uint32_t)__cvta_generic_to_shared(bar)), "h"(mask) : "memory");
    }
};

extern __shared__ __align__(1024) char swiftly_dyn_smem[];

// A body may declare WARP_BOUNDS = true: its CTAs are not whole warps (e.g. 10..28 threads),
// and the register budget below then counts the warps the hardware allocates for them.
template <class Body, class = void>
struct WarpBounds : std::false_type {};
template <class Body>
struct WarpBounds<Body, std::void_t<decltype(Body::WARP_BOUNDS)>>
    : std::integral_constant<bool, Body::WARP_BOUNDS> {};

// register budget: at least 512 resident threads per SM (<= 128 registers/thread).  Registers
// are allocated per warp, so a CTA of fewer than 32 threads costs a whole warp's registers:
// counted by thread, 512 / 16 = 32 such CTAs would hold 1024 threads' worth and cap them at 64.
template <class Body>
struct MinBlocks {
    static constexpr int ALLOC = WarpBounds<Body>::value ? (Body::THREADS + 31) / 32 * 32
                                                         : Body::THREADS;
    static constexpr int V = ALLOC >= 512 ? 1 : 512 / ALLOC;
};

template <class Body>
__global__ void __launch_bounds__(Body::THREADS, MinBlocks<Body>::V) kernel_entry(const Body body) {
    DeviceCtx ctx;
    ctx.tid = threadIdx.x;
    ctx.bid = blockIdx.x;
    ctx.nblocks = gridDim.x;
    ctx.smem = swiftly_dyn_smem;
    ctx.tmaps = nullptr;
    body(ctx);
}

// Kernels that use the TMA engine with tensor maps take the descriptors as a SEPARATE
// __grid_constant__ parameter (the TMA instructions need the descriptor's address in the
// parameter space); the body itself stays an ordinary by-value parameter -- measured: making
// the whole body __grid_constant__ changes code generation of the memory-bound line kernels
// for the worse (fewer registers, loads hoisted less far).
template <class Body>
__global__ void __launch_bounds__(Body::THREADS, MinBlocks<Body>::V)
    kernel_entry_maps(const Body body, const __grid_constant__ typename Body::Maps maps) {
    DeviceCtx ctx;
    ctx.tid = threadIdx.x;
    ctx.bid = blockIdx.x;
    ctx.nblocks = gridDim.x;
    ctx.smem = swiftly_dyn_smem;
    ctx.tmaps = &maps;
    body(ctx);
}

// launch helper: returns cudaError_t
template <class Body>
inline cudaError_t launch_body(const Body& body, int grid, size_t smem_bytes, cudaStream_t stream) {
    if (grid <= 0) return cudaSuccess;
    if (smem_bytes > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kernel_entry<Body>,
                                             cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)smem_bytes);
        if (e != cudaSuccess) return e;
    }
    kernel_entry<Body><<<grid, Body::THREADS, smem_bytes, stream>>>(body);
    return cudaGetLastError();
}

template <class Body>
inline cudaError_t launch_body_maps(const Body& body, const typename Body::Maps& maps, int grid,
                                    size_t smem_bytes, cudaStream_t stream) {
    if (grid <= 0) return cudaSuccess;
    if (smem_bytes > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kernel_entry_maps<Body>,
                                             cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)smem_bytes);
        if (e != cudaSuccess) return e;
    }
    kernel_entry_maps<Body><<<grid, Body::THREADS, smem_bytes, stream>>>(body, maps);
    return cudaGetLastError();
}

// kernel_entry_maps launched in clusters of Body::CLUSTER consecutive CTAs (grid a multiple of
// it).  Without a stream, only asks how many such clusters the device can hold at once
// (*clusters; 0: a cluster cannot be placed at all).
template <class Body>
inline cudaError_t launch_body_maps_cluster(const Body& body, const typename Body::Maps& maps,
                                            int grid, size_t smem_bytes, cudaStream_t stream,
                                            int* clusters) {
    cudaError_t e = cudaFuncSetAttribute(kernel_entry_maps<Body>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem_bytes);
    if (e != cudaSuccess) return e;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = Body::CLUSTER;
    attr.val.clusterDim.y = 1;
    attr.val.clusterDim.z = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid > 0 ? grid : Body::CLUSTER);
    cfg.blockDim = dim3(Body::THREADS);
    cfg.dynamicSmemBytes = smem_bytes;
    cfg.stream = stream;
    cfg.attrs = &attr;
    cfg.numAttrs = 1;
    if (clusters) return cudaOccupancyMaxActiveClusters(clusters, kernel_entry_maps<Body>, &cfg);
    if (grid <= 0) return cudaSuccess;
    return cudaLaunchKernelEx(&cfg, kernel_entry_maps<Body>, body, maps);
}
#endif

}  // namespace swiftly
