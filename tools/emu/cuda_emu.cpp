// cuda_emu.cpp — fiber scheduler and runtime stubs of the CPU emulation (see cuda_emu.h).  TEST TOOLING ONLY.
#include "cuda_emu.h"

#include <sys/mman.h>

#include <algorithm>
#include <chrono>
#include <numeric>
#include <random>
#include <mutex>
#include <vector>

namespace emu {

State g;
size_t stat_launches = 0, stat_threads = 0;

namespace {
constexpr size_t STACK_BYTES = 256 * 1024;
constexpr unsigned MAX_BLOCK = 1024;

struct WarpSlot {  // one barrier/exchange channel per distinct mask
    uint32_t mask = 0;
    uint64_t cnt[32] = {0};
    uint64_t val[2][32] = {{0}};
};
struct Warp {  // fixed storage: references stay valid while fibers are parked inside a collective
    WarpSlot slots[8];
    int n = 0;
    WarpSlot &slot(uint32_t mask) {
        for (int i = 0; i < n; i++)
            if (slots[i].mask == mask) return slots[i];
        if (n == 8) {
            std::fprintf(stderr, "emu: more than 8 distinct warp masks in one block\n");
            std::abort();
        }
        slots[n] = WarpSlot();
        slots[n].mask = mask;
        return slots[n++];
    }
};
struct Fiber {
    void *sp = nullptr;  // saved stack pointer while parked
    void *stack = nullptr;
    bool done = true;
    bool wait_block = false;  // parked in __syncthreads until bar_gen moves past wait_gen
    uint64_t wait_gen = 0;
    uint64_t progress = 0;    // sync points passed: lets the scheduler see whether a warp is still moving
};

void *sched_sp = nullptr;
std::vector<Fiber> fibers;
std::vector<Warp> warps;
const std::function<void()> *body = nullptr;
unsigned cur = 0, block_threads = 0, alive = 0;
unsigned bar_count = 0;
uint64_t bar_gen = 0;
bool in_kernel = false;
alignas(128) unsigned char smem_buf[232448];  // 227 KB: the per-CTA maximum on sm_90
}  // namespace
}  // namespace emu

// Minimal x86-64 System V context switch (callee-saved registers + stack pointer); glibc's swapcontext costs a
// sigprocmask system call per switch, which dominates a shuffle-heavy kernel.
extern "C" void emu_switch(void **save_sp, void *load_sp);
asm(R"(
    .text
    .globl emu_switch
    .type emu_switch,@function
emu_switch:
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
    .size emu_switch,.-emu_switch
)");

namespace emu {
namespace {

// EMU_SCHEDULE=fwd (default) | rev | rand:<seed> — the order in which blocks, warps and lanes get their turns.  Results
// of a correct kernel do not depend on it; running the tests under several schedules exposes order dependence.
struct Schedule {
    int mode;  // 0 forward, 1 reverse, 2 random
    unsigned seed;
};
Schedule schedule() {
    static const Schedule s = [] {
        const char *e = getenv("EMU_SCHEDULE");
        if (!e || !strcmp(e, "fwd")) return Schedule{0, 0};
        if (!strcmp(e, "rev")) return Schedule{1, 0};
        if (!strncmp(e, "rand", 4)) return Schedule{2, e[4] == ':' ? (unsigned)strtoul(e + 5, nullptr, 10) : 1u};
        std::fprintf(stderr, "emu: unknown EMU_SCHEDULE '%s'\n", e);
        std::abort();
    }();
    return s;
}

void fiber_entry() {
    (*body)();
    Fiber &f = fibers[cur];
    f.done = true;
    f.progress++;
    alive--;
    emu_switch(&f.sp, sched_sp);
    std::abort();  // a finished fiber is never resumed
}

void ensure_fibers(unsigned n) {
    if (fibers.size() < n) fibers.resize(n);
    for (unsigned i = 0; i < n; i++)
        if (!fibers[i].stack) {
            void *p = mmap(nullptr, STACK_BYTES, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS | MAP_STACK, -1, 0);
            if (p == MAP_FAILED) {
                std::fprintf(stderr, "emu: cannot allocate fiber stack\n");
                std::abort();
            }
            fibers[i].stack = p;
        }
}

void prepare(Fiber &f) {
    uintptr_t top = ((uintptr_t)f.stack + STACK_BYTES) & ~(uintptr_t)15;
    void **sp = (void **)top;
    *--sp = nullptr;                // return address of fiber_entry (never used)
    *--sp = (void *)fiber_entry;    // popped by emu_switch's ret
    for (int i = 0; i < 6; i++) *--sp = nullptr;  // rbp rbx r12 r13 r14 r15
    f.sp = sp;
    f.done = false;
    f.wait_block = false;
    f.progress = 0;
}

bool lane_exited(unsigned warp, unsigned lane) {
    unsigned t = warp * 32 + lane;
    return t >= block_threads || fibers[t].done;
}
}  // namespace

void *dynamic_smem(size_t bytes) {
    if (bytes > sizeof smem_buf) {
        std::fprintf(stderr, "emu: %zu bytes of dynamic shared memory requested (max %zu)\n", bytes, sizeof smem_buf);
        std::abort();
    }
    return smem_buf;
}
void *smem_base() { return smem_buf; }

void yield() {
    if (!in_kernel) return;
    unsigned me = cur;
    emu_switch(&fibers[me].sp, sched_sp);
    g.tid = uint3{me, 0, 0};
}

void sync_block() {
    Fiber &f = fibers[cur];
    f.wait_gen = bar_gen;
    f.wait_block = true;
    bar_count++;
    while (bar_gen == f.wait_gen) yield();
    f.wait_block = false;
    f.progress++;
}

void sync_warp(uint32_t mask) {
    unsigned w = g.tid.x >> 5, lane = g.tid.x & 31;
    WarpSlot &s = warps[w].slot(mask);
    uint64_t my = ++s.cnt[lane];
    for (;;) {
        bool all = true;
        for (unsigned l = 0; l < 32 && all; l++)
            if ((mask >> l & 1) && l != lane && s.cnt[l] < my && !lane_exited(w, l)) all = false;
        if (all) break;
        yield();
    }
    fibers[w * 32 + lane].progress++;
}

uint64_t warp_exchange(uint32_t mask, uint64_t mine, int src_lane, bool *src_valid) {
    unsigned w = g.tid.x >> 5, lane = g.tid.x & 31;
    WarpSlot &s = warps[w].slot(mask);
    unsigned parity = (unsigned)((s.cnt[lane] + 1) & 1);
    s.val[parity][lane] = mine;
    sync_warp(mask);
    // the source took part iff it reached this exchange (it may have run on and exited since: its value stays put)
    const uint64_t my = s.cnt[lane];
    *src_valid = src_lane >= 0 && src_lane < 32 && (mask >> src_lane & 1) && s.cnt[src_lane] >= my;
    return *src_valid ? s.val[parity][src_lane] : mine;
}

uint64_t warp_reduce_or(uint32_t mask, uint64_t mine) {
    unsigned w = g.tid.x >> 5, lane = g.tid.x & 31;
    WarpSlot &s = warps[w].slot(mask);
    unsigned parity = (unsigned)((s.cnt[lane] + 1) & 1);
    s.val[parity][lane] = mine;
    sync_warp(mask);
    const uint64_t my = s.cnt[lane];
    uint64_t r = 0;
    for (unsigned l = 0; l < 32; l++)
        if ((mask >> l & 1) && s.cnt[l] >= my) r |= s.val[parity][l];
    return r;
}

void run_grid(unsigned grid, unsigned block, const std::function<void()> &thread_body) {
    if (block == 0 || block > MAX_BLOCK || grid == 0) {
        std::fprintf(stderr, "emu: bad launch configuration <<<%u, %u>>>\n", grid, block);
        std::abort();
    }
    static std::mutex launch_mu;  // the scheduler state is global: launches from several host threads take turns
    std::lock_guard<std::mutex> launch_guard(launch_mu);
    if (in_kernel) {
        std::fprintf(stderr, "emu: nested launch\n");
        std::abort();
    }
    stat_launches++;
    stat_threads += (size_t)grid * block;
    ensure_fibers(block);
    body = &thread_body;
    block_threads = block;
    g.bdim = dim3(block);
    g.gdim = dim3(grid);
    in_kernel = true;
    const unsigned n_warps = (block + 31) / 32;
    const Schedule sched = schedule();
    std::vector<unsigned> block_order(grid), lane_order(32), warp_order(n_warps);
    std::iota(block_order.begin(), block_order.end(), 0u);
    std::iota(lane_order.begin(), lane_order.end(), 0u);
    std::iota(warp_order.begin(), warp_order.end(), 0u);
    if (sched.mode == 1) {
        std::reverse(block_order.begin(), block_order.end());
        std::reverse(lane_order.begin(), lane_order.end());
        std::reverse(warp_order.begin(), warp_order.end());
    } else if (sched.mode == 2) {
        std::mt19937 rng(sched.seed + (unsigned)stat_launches * 7919u);
        std::shuffle(block_order.begin(), block_order.end(), rng);
        std::shuffle(lane_order.begin(), lane_order.end(), rng);
        std::shuffle(warp_order.begin(), warp_order.end(), rng);
    }
    for (unsigned bi = 0; bi < grid; bi++) {
        const unsigned b = block_order[bi];
        g.bid = uint3{b, 0, 0};
        warps.assign(n_warps, Warp());
        bar_count = 0;
        alive = block;
        for (unsigned t = 0; t < block; t++) prepare(fibers[t]);
        unsigned stalled_rounds = 0;
        while (alive) {
            bool any_progress = false;
            for (unsigned wi = 0; wi < n_warps; wi++) {
                const unsigned w = warp_order[wi];
                unsigned lo = w * 32, hi = lo + 32 < block ? lo + 32 : block;
                for (;;) {  // keep a warp going while its lanes still pass sync points or finish
                    uint64_t before = 0, after = 0;
                    bool ran = false;
                    for (unsigned t = lo; t < hi; t++) before += fibers[t].progress;
                    for (unsigned li = 0; li < 32; li++) {
                        const unsigned t = lo + lane_order[li];
                        if (t >= hi) continue;
                        Fiber &f = fibers[t];
                        if (f.done || (f.wait_block && bar_gen == f.wait_gen)) continue;
                        cur = t;
                        g.tid = uint3{t, 0, 0};
                        emu_switch(&sched_sp, f.sp);
                        ran = true;
                        if (bar_count && bar_count >= alive) {  // all live threads arrived (exited ones count as arrived)
                            bar_count = 0;
                            bar_gen++;
                        }
                    }
                    for (unsigned t = lo; t < hi; t++) after += fibers[t].progress;
                    if (after != before) any_progress = true;
                    if (!ran || after == before) break;
                }
            }
            if (bar_count && bar_count >= alive) {
                bar_count = 0;
                bar_gen++;
                any_progress = true;
            }
            stalled_rounds = any_progress ? 0 : stalled_rounds + 1;
            if (stalled_rounds > 4) {
                std::fprintf(stderr, "emu: deadlock in block %u (a barrier or warp collective not reached by all of its threads)\n", b);
                std::abort();
            }
        }
    }
    in_kernel = false;
    body = nullptr;
}

}  // namespace emu

// ------------------------------------------------------------------------------------------------ runtime stubs
struct emuStream { int dummy; };
struct emuEvent { std::chrono::steady_clock::time_point t; };

cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return cudaSuccess; }
cudaError_t cudaSetDevice(int) { return cudaSuccess; }
cudaError_t cudaGetDevice(int *d) { *d = 0; return cudaSuccess; }
cudaError_t cudaGetLastError() { return cudaSuccess; }
const char *cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : e == cudaErrorMemoryAllocation ? "out of memory" : "emulated error"; }
cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
cudaError_t cudaDeviceGetAttribute(int *v, cudaDeviceAttr a, int) {
    // two "SMs": persistent grids get more than one block, so grid-stride loops are exercised
    *v = a == cudaDevAttrMultiProcessorCount ? 2 : 0;
    return cudaSuccess;
}
cudaError_t cudaMalloc(void **p, size_t bytes) {
    *p = nullptr;
    if (posix_memalign(p, 256, bytes ? bytes : 1)) return cudaErrorMemoryAllocation;
    memset(*p, 0xCD, bytes);  // device memory is not zeroed: make reliance on that visible
    return cudaSuccess;
}
cudaError_t cudaFree(void *p) { free(p); return cudaSuccess; }
cudaError_t cudaMallocHost(void **p, size_t bytes) {
    *p = nullptr;
    return posix_memalign(p, 256, bytes ? bytes : 1) ? cudaErrorMemoryAllocation : cudaSuccess;
}
cudaError_t cudaFreeHost(void *p) { free(p); return cudaSuccess; }
cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { if (n) memmove(d, s, n); return cudaSuccess; }
cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t) { if (n) memmove(d, s, n); return cudaSuccess; }
cudaError_t cudaMemset(void *d, int v, size_t n) { if (n) memset(d, v, n); return cudaSuccess; }
cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t) { if (n) memset(d, v, n); return cudaSuccess; }
cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = new emuStream{0}; return cudaSuccess; }
cudaError_t cudaStreamCreateWithPriority(cudaStream_t *s, unsigned, int) { *s = new emuStream{0}; return cudaSuccess; }
cudaError_t cudaDeviceGetPCIBusId(char *b, int n, int) { if (n > 0) b[0] = 0; return cudaErrorInvalidValue; }
cudaError_t cudaDeviceGetStreamPriorityRange(int *lo, int *hi) { if (lo) *lo = 0; if (hi) *hi = -5; return cudaSuccess; }
cudaError_t cudaStreamCreate(cudaStream_t *s) { *s = new emuStream{0}; return cudaSuccess; }
cudaError_t cudaStreamDestroy(cudaStream_t s) { if (s != cudaStreamLegacy) delete s; return cudaSuccess; }
cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = new emuEvent{std::chrono::steady_clock::now()}; return cudaSuccess; }
cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { return cudaEventCreate(e); }
cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t) { e->t = std::chrono::steady_clock::now(); return cudaSuccess; }
cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t a, cudaEvent_t b) {
    *ms = std::chrono::duration<float, std::milli>(b->t - a->t).count();
    return cudaSuccess;
}
