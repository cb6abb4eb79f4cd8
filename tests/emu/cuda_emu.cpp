// TEST INFRASTRUCTURE ONLY: fiber scheduler for tests/emu/cuda_emu.h
#include "cuda_emu.h"
#include <stdexcept>

thread_local EmuState emu_cur;

namespace {
// Persistent fibers: one per thread slot of a block, created once (makecontext) and reused by every block of every launch.  All
// later switches are _setjmp / _longjmp pairs: unlike swapcontext / getcontext they make no system call (glibc saves and restores the
// signal mask there), which dominated the run time of launches with many short threads.
struct Fiber {
    ucontext_t ctx;
    jmp_buf jb;
    unsigned char* stack = nullptr;
    EmuState st;
    bool done = false;
    bool created = false;
};
const size_t STACK = 128 * 1024;
thread_local Fiber fiber_pool[1024];                    // a block has at most 1024 threads
thread_local jmp_buf sched_jb;
thread_local Fiber* running = nullptr;
thread_local const std::function<void()>* cur_body = nullptr;

void fiber_main() {
    for (;;) {                                          // one iteration per (launch, block) this slot takes part in
        (*cur_body)();
        running->done = true;
        if (!_setjmp(running->jb)) _longjmp(sched_jb, 1);      // parked until the next block resumes this slot
    }
}

// scheduler side: run fiber f until it yields or finishes
void resume(Fiber& f) {
    running = &f;
    emu_cur = f.st;
    if (_setjmp(sched_jb)) return;                      // the fiber came back
    if (f.created) _longjmp(f.jb, 1);
    f.created = true;
    if (!f.stack) f.stack = (unsigned char*)malloc(STACK);
    getcontext(&f.ctx);
    f.ctx.uc_stack.ss_sp = f.stack;
    f.ctx.uc_stack.ss_size = STACK;
    f.ctx.uc_link = nullptr;
    makecontext(&f.ctx, (void (*)())fiber_main, 0);
    setcontext(&f.ctx);                                 // first entry of this slot; never returns here
}
}  // namespace

// one scheduling step: give the other fibers of the block a turn
void emu_yield() {
    Fiber* f = running;
    f->st = emu_cur;
    if (!_setjmp(f->jb)) _longjmp(sched_jb, 1);
    emu_cur = f->st;
}

// block barrier: a real arrival count (threads that already exited count as arrived, as on the GPU), so that code
// between two barriers may yield a different number of times in different warps (warp shuffles, see below)
static thread_local size_t bar_arrived = 0, bar_generation = 0, bar_live = 0;
static void bar_release_if_complete() {
    if (bar_live > 0 && bar_arrived >= bar_live) { bar_arrived = 0; ++bar_generation; }
}
void emu_syncthreads() {
    const size_t gen = bar_generation;
    ++bar_arrived;
    bar_release_if_complete();
    while (bar_generation == gen) emu_yield();
}

static double shfl_slots[2][4096];
static unsigned char shfl_parity[4096];
double emu_shfl_exchange(double v, int src_lane) {
    // two slot sets used alternately: a lane overwrites set p again only in its call after next, i.e. after the yield of the
    // call in between, by which every lane of the warp has finished reading set p -- one yield per exchange is enough
    const unsigned tid = emu_cur.tid.x;            // 1-D blocks only
    const unsigned p = shfl_parity[tid] ^= 1;
    shfl_slots[p][tid] = v;
    emu_yield();                                   // every lane of the warp has published (lanes run in lockstep)
    return shfl_slots[p][(tid & ~31u) + (unsigned)src_lane];
}

// cp.async: one queue per thread slot of the running block.  A copy belongs to the open group (numbered by the count of groups
// committed before it); cp.async.wait_group n lands, in issue order, the copies of every group but the n most recent.  The source is
// read at landing time too: the kernels never write what they prefetch while the copy is in flight.
namespace {
struct CpCopy { void* dst; const void* src; size_t bytes; size_t group; };
struct CpQueue {
    std::vector<CpCopy> copies;
    size_t head = 0, committed = 0;
    void reset() { copies.clear(); head = 0; committed = 0; }
};
thread_local CpQueue cp_queues[1024];
bool cp_late() {
    static const bool late = [] {
        const char* e = getenv("DB_EMU_CP");
        if (!e || !strcmp(e, "late")) return true;
        if (!strcmp(e, "early")) return false;
        fprintf(stderr, "DB_EMU_CP=%s: expected 'late' or 'early'\n", e);
        abort();
    }();
    return late;
}
CpQueue& cp_queue() {
    const EmuState& s = emu_cur;
    return cp_queues[s.tid.x + s.bdim.x * (s.tid.y + s.bdim.y * s.tid.z)];
}
}  // namespace

void emu_cp_async(void* dst, const void* src, size_t bytes) {
    if (!cp_late()) { std::memcpy(dst, src, bytes); return; }
    CpQueue& q = cp_queue();
    q.copies.push_back({dst, src, bytes, q.committed});
}

void emu_cp_commit() { ++cp_queue().committed; }

void emu_cp_wait(int n) {
    CpQueue& q = cp_queue();
    if (q.committed <= (size_t)n) return;
    const size_t retire = q.committed - (size_t)n;        // groups 0 .. retire - 1 complete
    while (q.head < q.copies.size() && q.copies[q.head].group < retire) {
        const CpCopy& c = q.copies[q.head++];
        std::memcpy(c.dst, c.src, c.bytes);
    }
    if (q.head == q.copies.size()) { q.copies.clear(); q.head = 0; }
}

void emu_launch(dim3 grid, dim3 block, size_t smem, const std::function<void()>& body) {
    const size_t nthreads = (size_t)block.x * block.y * block.z;
    // the launch limits of the real device (sm_90): a launch that violates them fails on the GPU with "invalid configuration
    // argument" while a host loop would just run zero or too many iterations
    if (grid.x == 0 || grid.y == 0 || grid.z == 0 || nthreads == 0 || nthreads > 1024 || block.z > 64 || grid.y > 65535 || grid.z > 65535 ||
        smem > 227 * 1024) {
        fprintf(stderr, "emu_launch: invalid CUDA launch configuration grid=(%u,%u,%u) block=(%u,%u,%u) smem=%zu\n",
                grid.x, grid.y, grid.z, block.x, block.y, block.z, smem);
        abort();
    }
    std::vector<unsigned char> shared(smem + 64);
    Fiber* fibers = fiber_pool;
    cur_body = &body;
    static const bool reverse_blocks = [] { const char* e = getenv("DB_EMU_ORDER"); return e && e[0] == 'r'; }();
    for (unsigned bzi = 0; bzi < grid.z; ++bzi)
    for (unsigned byi = 0; byi < grid.y; ++byi)
    for (unsigned bxi = 0; bxi < grid.x; ++bxi) {
        // blocks of a grid run one after the other here; on the GPU their order is arbitrary: reversed with DB_EMU_ORDER=reverse
        const unsigned bz = reverse_blocks ? grid.z - 1 - bzi : bzi, by = reverse_blocks ? grid.y - 1 - byi : byi,
                       bx = reverse_blocks ? grid.x - 1 - bxi : bxi;
        std::memset(shared.data(), 0xA5, shared.size());   // poison shared memory
        std::memset(shfl_parity, 0, sizeof(shfl_parity));
        // copies still pending when a thread of the previous block exited never land in this block's shared memory
        for (size_t t = 0; t < nthreads; ++t) cp_queues[t].reset();
        size_t i = 0;
        for (unsigned tz = 0; tz < block.z; ++tz)
        for (unsigned ty = 0; ty < block.y; ++ty)
        for (unsigned tx = 0; tx < block.x; ++tx, ++i) {
            Fiber& f = fibers[i];
            f.done = false;
            f.st.tid = {tx, ty, tz}; f.st.bid = {bx, by, bz}; f.st.bdim = block; f.st.gdim = grid;
            f.st.smem = shared.data();
        }
        size_t remaining = nthreads;
        bar_arrived = 0; bar_live = nthreads;
        // DB_EMU_ORDER=reverse: the threads of a block take their turns in descending order.  Code that is correct only because a
        // lower-numbered thread happens to run first (a missing __syncthreads / __syncwarp) passes in one order and fails in the other.
        static const bool reverse_order = [] { const char* e = getenv("DB_EMU_ORDER"); return e && e[0] == 'r'; }();
        while (remaining) {
            size_t finished_this_round = 0, waiting = 0;
            for (size_t fi = 0; fi < nthreads; ++fi) {
                Fiber& f = fibers[reverse_order ? nthreads - 1 - fi : fi];
                if (f.done) continue;
                resume(f);
                if (f.done) { ++finished_this_round; --bar_live; bar_release_if_complete(); } else { ++waiting; }
            }
            remaining -= finished_this_round;
            if (finished_this_round && waiting) {
                // some threads exited while others wait at a barrier: allowed in CUDA only if exited threads
                // never reach the barrier; continue scheduling the waiting ones.
            }
        }
    }
    running = nullptr;
}
