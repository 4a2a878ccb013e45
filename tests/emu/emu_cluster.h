// TEST TOOLING ONLY -- host emulation of thread block clusters, on top of emu_runtime.h.
//
// The CTAs of one cluster run together: every thread of every CTA is a fibre of one round-robin
// scheduler (a sweep runs each live thread to its next wait, CTA rank 0 first).  A kernel body
// launched through launch_body_maps_cluster gets a ClusterHostCtx: the HostCtx of its CTA (CTA
// barriers, named barriers and the bulk-copy accounting of emu_runtime.h, per CTA) plus the
// cluster operations of DeviceCtx (common.cuh):
//   * cluster_rank, cluster_sync (a barrier over every thread of the cluster);
//   * peer_st / peer_atomic_add: distributed shared memory, an address of the caller's shared
//     memory mapped to the same offset in CTA `rank`;
//   * tx_expect_peer: arming the bulk-copy barrier of CTA `rank`;
//   * tensor_load_mc / tx_copy_mc: a multicast, delivered to each destination CTA's shared
//     memory and counted against that CTA's barrier.
// Reported as protocol errors (the process aborts), like the barrier errors of emu_runtime.h:
//   * a wait on a cluster barrier while a thread of the cluster has exited: it cannot complete;
//   * a store, atomic, barrier arming or multicast into the shared memory of an exited CTA;
//   * a multicast into a CTA whose barrier is not armed or that delivers more bytes than that
//     CTA's phase was armed with (the accounting of emu_runtime.h, per destination CTA);
//   * a grid that is not whole clusters is refused (cudaErrorInvalidValue), as by the driver.
#pragma once

#include "emu_runtime.h"

namespace swiftly {

struct EmuCluster;

struct ClusterHostCtx : HostCtx {
    EmuCluster* cl;
    int rank;
    int cluster_rank() const { return rank; }
    inline void cluster_sync() const;
    inline void peer_st(double2* p, int r, double2 v) const;
    inline int peer_atomic_add(int* p, int r, int v) const;
    inline void tx_expect_peer(uint64_t* bar, int r, uint32_t bytes) const;
    inline void tensor_load_mc(void* smem_dst, const void* map, int c1, int c2, uint64_t* bar,
                               uint16_t mask) const;
    inline void tx_copy_mc(void* smem_dst, const void* src, uint32_t bytes, uint64_t* bar,
                           uint16_t mask) const;
    // the HostCtx of CTA `r` (its shared memory, its barriers), which must still be running
    inline HostCtx peer(int r, const char* what) const;
    template <class T>
    T* map(T* p, const HostCtx& to) const {
        const size_t off = (size_t)((const char*)p - smem);
        return (T*)(to.smem + off);
    }
};

struct EmuCluster {
    static constexpr int MAX = 8;
    int size;
    EmuBlock blk[MAX];
    char* smem[MAX];
    std::vector<ClusterHostCtx> cctx[MAX];
    void (*entry)(void*, ClusterHostCtx&);
    void* body;
    int cur_rank, cur_t;
    int arrived;  // cluster barrier
    unsigned gen;
};

static EmuCluster* g_emu_cluster = nullptr;

static inline void emu_cluster_error(const HostCtx& c, const char* what, int r) {
    fprintf(stderr, "swiftly emulator: cluster PROTOCOL error in block %d, thread %d: %s (CTA rank %d)\n",
            c.bid, c.tid, what, r);
    abort();
}

static inline bool emu_cta_exited(const EmuBlock& b) {
    for (char d : b.done)
        if (!d) return false;
    return true;
}

inline HostCtx ClusterHostCtx::peer(int r, const char* what) const {
    if (r < 0 || r >= cl->size) emu_cluster_error(*this, "rank outside the cluster", r);
    if (emu_cta_exited(cl->blk[r])) emu_cluster_error(*this, what, r);
    HostCtx pc = *this;
    pc.blk = &cl->blk[r];
    pc.smem = cl->smem[r];
    return pc;
}

inline void ClusterHostCtx::cluster_sync() const {
    int total = 0;
    for (int r = 0; r < cl->size; ++r) total += cl->blk[r].nthreads;
    const unsigned g = cl->gen;
    if (++cl->arrived == total) {
        cl->arrived = 0;
        ++cl->gen;
        ++blk->progress;
        yield();  // who runs first after the barrier is up to the sweep, as for the others
        return;
    }
    while (cl->gen == g) {
        for (int r = 0; r < cl->size; ++r)
            for (char d : cl->blk[r].done)
                if (d) emu_cluster_error(*this, "wait on a cluster barrier that cannot complete "
                                                "(a thread of the cluster has exited)", r);
        yield();
    }
}

inline void ClusterHostCtx::peer_st(double2* p, int r, double2 v) const {
    const HostCtx pc = peer(r, "store into the shared memory of a CTA which has exited");
    *map(p, pc) = v;
}

inline int ClusterHostCtx::peer_atomic_add(int* p, int r, int v) const {
    const HostCtx pc = peer(r, "atomic on the shared memory of a CTA which has exited");
    int* q = map(p, pc);
    const int prev = *q;
    *q = prev + v;
    return prev;
}

inline void ClusterHostCtx::tx_expect_peer(uint64_t* bar, int r, uint32_t bytes) const {
    const HostCtx pc = peer(r, "barrier arming in a CTA which has exited");
    pc.tx_expect(map(bar, pc), bytes);
}

inline void ClusterHostCtx::tensor_load_mc(void* smem_dst, const void* m, int c1, int c2,
                                           uint64_t* bar, uint16_t mask) const {
    for (int r = 0; r < cl->size; ++r)
        if (mask >> r & 1) {
            const HostCtx pc = peer(r, "multicast into a CTA which has exited");
            pc.tensor_load(map((char*)smem_dst, pc), m, c1, c2, map(bar, pc));
        }
}

inline void ClusterHostCtx::tx_copy_mc(void* smem_dst, const void* src, uint32_t bytes,
                                       uint64_t* bar, uint16_t mask) const {
    for (int r = 0; r < cl->size; ++r)
        if (mask >> r & 1) {
            const HostCtx pc = peer(r, "multicast into a CTA which has exited");
            pc.tx_copy(map((char*)smem_dst, pc), src, bytes, map(bar, pc));
        }
}

static void emu_cluster_trampoline() {
    EmuCluster* cl = g_emu_cluster;
    const int r = cl->cur_rank, t = cl->cur_t;
    cl->entry(cl->body, cl->cctx[r][t]);
    cl->blk[r].done[t] = 1;
    ++cl->blk[r].progress;
}

template <class Body>
static void emu_cluster_entry(void* body, ClusterHostCtx& ctx) {
    (*(const Body*)body)(ctx);
}

// as on the device (common.cuh); an emulated H100 holds one CTA of these kernels per SM, so
// 132 / CLUSTER clusters
template <class Body>
inline cudaError_t launch_body_maps_cluster(const Body& body, const typename Body::Maps& maps,
                                            int grid, size_t smem_bytes, cudaStream_t,
                                            int* clusters) {
    const int C = Body::CLUSTER, T = Body::THREADS;
    static_assert(Body::CLUSTER >= 1 && Body::CLUSTER <= EmuCluster::MAX, "cluster size");
    if (clusters) {
        *clusters = 132 / C;
        return cudaSuccess;
    }
    if (grid <= 0) return cudaSuccess;
    if (grid % C) return cudaErrorInvalidValue;
    const size_t STACK = 256 * 1024;
    EmuCluster* cl = new EmuCluster();
    cl->size = C;
    cl->entry = &emu_cluster_entry<Body>;
    cl->body = (void*)&body;
    for (int r = 0; r < C; ++r) {
        EmuBlock& b = cl->blk[r];
        b.ctxs.resize(T);
        b.stacks.resize(T);
        b.done.resize(T);
        b.nthreads = T;
        for (int t = 0; t < T; ++t) b.stacks[t] = (char*)malloc(STACK);
        cl->smem[r] = (char*)malloc(smem_bytes + 64);
        cl->cctx[r].resize(T);
    }
    for (int bid0 = 0; bid0 < grid; bid0 += C) {
        cl->arrived = 0;
        cl->gen = 0;
        for (int r = 0; r < C; ++r) {
            EmuBlock& b = cl->blk[r];
            memset(cl->smem[r], 0xA5, smem_bytes + 64);  // poison: uninitialised reads show up
            for (int t = 0; t < T; ++t) {
                getcontext(&b.ctxs[t]);
                b.ctxs[t].uc_stack.ss_sp = b.stacks[t];
                b.ctxs[t].uc_stack.ss_size = STACK;
                b.ctxs[t].uc_link = &b.main_ctx;
                makecontext(&b.ctxs[t], (void (*)())emu_cluster_trampoline, 0);
                b.done[t] = 0;
                ClusterHostCtx& c = cl->cctx[r][t];
                c.tid = t;
                c.bid = bid0 + r;
                c.nblocks = grid;
                c.smem = cl->smem[r];
                c.tmaps = &maps;
                c.blk = &b;
                c.cl = cl;
                c.rank = r;
            }
            b.tx.clear();
            for (int i = 0; i < 16; ++i) {
                b.bar_arrived[i] = 0;
                b.bar_gen[i] = 0;
            }
            b.progress = 0;
        }
        auto progress = [&]() {
            unsigned long p = 0;
            for (int r = 0; r < C; ++r) p += cl->blk[r].progress;
            return p;
        };
        bool any = true;
        int idle_sweeps = 0;
        while (any) {
            any = false;
            const unsigned long before = progress();
            for (int r = 0; r < C; ++r) {
                EmuBlock& b = cl->blk[r];
                for (int t = 0; t < T; ++t) {
                    if (b.done[t]) continue;
                    g_emu_cluster = cl;
                    cl->cur_rank = r;
                    cl->cur_t = t;
                    swapcontext(&b.main_ctx, &b.ctxs[t]);
                    if (!b.done[t]) any = true;
                }
            }
            idle_sweeps = (any && progress() == before) ? idle_sweeps + 1 : 0;
            if (idle_sweeps >= 2) {
                fprintf(stderr, "swiftly emulator: barrier DEADLOCK in the cluster of blocks %d .. %d "
                                "(%d threads at the cluster barrier)\n", bid0, bid0 + C - 1,
                        cl->arrived);
                abort();
            }
        }
    }
    for (int r = 0; r < C; ++r) {
        free(cl->smem[r]);
        for (int t = 0; t < T; ++t) free(cl->blk[r].stacks[t]);
    }
    delete cl;
    return cudaSuccess;
}

}  // namespace swiftly
