// engine.h — context and scratch-arena definitions shared by the translation units of libb200trie.so.
#pragma once
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <utility>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/b200trie.h"
#include "pinned_pool.h"

// ------------------------------------------------------------------------------------------------ device memory
// One block of device memory, charged to the byte counter of its owner (b200_ctx::dev_bytes, or the `bytes` of a trie or
// state).  Released, and taken off that counter, by reset(), by the destructor, or when a move overwrites it.  An owner
// declares its counter before the buffers charged to it: members are destroyed in reverse order.  The caller makes sure
// no queued work still uses a block it releases.  Only grow() allocates.
struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
    uint64_t *owner = nullptr;  // the counter `cap` is charged to

    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    DevBuf(DevBuf &&o) noexcept : p(o.p), cap(o.cap), owner(o.owner) {
        o.p = nullptr;
        o.cap = 0;
    }
    DevBuf &operator=(DevBuf &&o) noexcept {
        if (this != &o) {
            reset();
            std::swap(p, o.p);
            std::swap(cap, o.cap);
            owner = o.owner;
        }
        return *this;
    }
    ~DevBuf() { reset(); }
    void reset() {
        if (p) {
            cudaFree(p);
            *owner -= cap;
        }
        p = nullptr;
        cap = 0;
    }
    // takes over `src`'s block (releasing this one's) and charges it to `counter`: a buffer handed to another owner
    void take(DevBuf &src, uint64_t *counter) {
        *this = std::move(src);
        if (p) {
            *owner -= cap;
            *counter += cap;
        }
        owner = counter;
    }
};

// ------------------------------------------------------------------------------------------------ context

struct b200_ctx {
    int device = 0;
    cudaStream_t own_stream = nullptr, stream = nullptr;
    cudaStream_t copy_streams[3] = {nullptr, nullptr, nullptr};
    // structure pass of a build (sorts, scans, flags: memory / latency bound) runs here, next to the ALU-bound leaf pass
    // on `stream`; highest priority, so that its short kernels get the SM slots the leaf pass frees
    cudaStream_t aux_stream = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    std::vector<cudaEvent_t> chunk_events;
    std::mutex mu;
    std::mutex err_mu;  // guards err: argument checks report errors before they take `mu`
    std::string err;
    uint64_t dev_bytes = 0;
    unsigned launches = 0;
    b200_stats stats{};
    bool stats_pending = false;
    bool stats_wavefront = false;  // branches_added of the last build comes from the wavefront's node counter
    uint64_t extra_blocks = 0;     // rate blocks beyond the first of the branch nodes built since reset_build_state
    bool extra_blocks_valid = false;  // every node of this call went through build_forest's class histogram
    // scratch (grow-only)
    DevBuf Lp, nibs, leaf_ref, leaf_meta, S, E, iota, depth_sorted, gap_sorted, head, node_start,
        node_ref, node_meta, node_l, node_r, node_masks, cub_temp, small, sroots, buckets;
    DevBuf upd_flags, upd_nh, upd_ids, upd_prefix, upd_key, upd_key2, upd_ids2;
    DevBuf sort_ka, sort_kb, sort_ia, sort_flag, sort_perm, sort_out;
    DevBuf sort_aux[4];  // composite sort: sorted address digests, their permutation, head flags / dense ranks, rank by address
    DevBuf node_key, node_key2, node_ids, node_order;
    DevBuf ord_keys, ord_knib, ord_item, ord_sched, ord_sched2, ord_pos, ord_order;  // ordered tries (eng_ordered.inl)
    DevBuf sl[29];  // stateless roots (eng_stateless.inl) and overlay roots (eng_overlay.inl)
    // staging for host-pointer entry points
    DevBuf in_a, in_b, in_c, in_d, in_e, out_a, chunk_in[3], chunk_out[3];
    void *pinned_small = nullptr;  // 4 KiB page-locked readback area
    // B200_PHASE_TIMING=1 (development aid): CUDA events at the phase boundaries of a build, reported by b200_sync on stderr
    bool phase_timing = false;
    std::vector<std::pair<const char *, cudaEvent_t>> phases;
    std::vector<cudaEvent_t> phase_pool;
};

inline void phase_mark(b200_ctx *c, const char *name) {
    if (!c->phase_timing) return;
    cudaEvent_t ev = nullptr;
    if (!c->phase_pool.empty()) {
        ev = c->phase_pool.back();
        c->phase_pool.pop_back();
    } else if (cudaEventCreate(&ev) != cudaSuccess) {
        return;
    }
    cudaEventRecord(ev, c->stream);
    c->phases.emplace_back(name, ev);
}
inline void phase_report(b200_ctx *c) {  // after a stream synchronize
    if (c->phases.size() > 1) {
        float total = 0;
        cudaEventElapsedTime(&total, c->phases.front().second, c->phases.back().second);
        fprintf(stderr, "[b200 phases] total %.3f ms:", total);
        for (size_t i = 1; i < c->phases.size(); i++) {
            float ms = 0;
            cudaEventElapsedTime(&ms, c->phases[i - 1].second, c->phases[i].second);
            fprintf(stderr, " %s %.3f", c->phases[i].first, ms);
        }
        fprintf(stderr, "\n");
    }
    for (auto &p : c->phases) c->phase_pool.push_back(p.second);
    c->phases.clear();
}

inline int32_t fail(b200_ctx *c, int32_t code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (c) {
        std::lock_guard<std::mutex> g(c->err_mu);
        c->err = buf;
    }
    return code;
}

#define CU(call)                                                                                              \
    do {                                                                                                      \
        cudaError_t e__ = (call);                                                                             \
        if (e__ != cudaSuccess)                                                                               \
            return fail(c, e__ == cudaErrorMemoryAllocation ? B200_ERR_OOM : B200_ERR_CUDA, "%s: %s (%s:%d)", \
                        #call, cudaGetErrorString(e__), __FILE__, __LINE__);                                  \
    } while (0)

// Every device allocation: if `b` holds fewer than `need` bytes, it gets a new block of `want` bytes charged to *counter,
// filled with the byte `fill` (>= 0) and holding the first `keep` bytes of the old block.  With nothing to keep the old
// block is released first, so that the two never coexist.  On failure `b` is either unchanged or empty, and every
// counter matches what is allocated.
inline int32_t grow(b200_ctx *c, uint64_t *counter, DevBuf &b, size_t need, size_t want, size_t keep = 0, int fill = -1) {
    if (need <= b.cap) return B200_OK;
    if (c->phase_timing) fprintf(stderr, "[b200 grow] %zu -> %zu bytes (keep %zu)\n", b.cap, want, keep);
    if (b.p && !keep) {
        CU(cudaStreamSynchronize(c->stream));  // the block may still be in use by queued work
        b.reset();
    }
    void *p = nullptr;
    CU(cudaMalloc(&p, want));
    DevBuf nb;
    nb.p = p;
    nb.cap = want;
    nb.owner = counter;
    *counter += want;
    if (fill >= 0) CU(cudaMemsetAsync(p, fill, want, c->stream));
    if (b.p) {
        CU(cudaMemcpyAsync(p, b.p, keep, cudaMemcpyDeviceToDevice, c->stream));
        CU(cudaStreamSynchronize(c->stream));
    }
    b = std::move(nb);
    return B200_OK;
}
// size rules: the context's scratch takes 1/8 slack, so that slowly growing inputs do not re-allocate every call;
// resident tries and arena capacity are sized to fit
inline size_t ctx_cap(size_t bytes) { return bytes + bytes / 8 + 256; }
inline int32_t ensure(b200_ctx *c, DevBuf &b, size_t bytes) { return grow(c, &c->dev_bytes, b, bytes, ctx_cap(bytes)); }
inline int32_t grow_fit(b200_ctx *c, uint64_t *counter, DevBuf &b, size_t bytes, size_t keep = 0, int fill = -1) {
    return grow(c, counter, b, bytes, bytes + 256, keep, fill);
}
#define ENSURE(buf, bytes)                                   \
    do {                                                     \
        int32_t r__ = ensure(c, c->buf, (size_t)(bytes));    \
        if (r__ != B200_OK) return r__;                      \
    } while (0)
#define TRY(expr)                         \
    do {                                  \
        int32_t r__ = (expr);             \
        if (r__ != B200_OK) return r__;   \
    } while (0)

