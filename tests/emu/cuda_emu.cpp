// TEST INFRASTRUCTURE ONLY: fiber scheduler for tests/emu/cuda_emu.h
#include "cuda_emu.h"
#include <cstdarg>
#include <cstdint>
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
    const char* wait_what = nullptr;                    // set when the fiber last yielded from an emulated wait (deadlock detection)
    const void* wait_on = nullptr;
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

// every change of barrier or copy-queue state counts here: a scheduling round in which it stays put while every live fiber
// waits is a deadlock
static thread_local size_t emu_progress = 0;
// a yield from inside an emulated wait: records what the fiber waits for
static void emu_wait_yield(const char* what, const void* on) {
    running->wait_what = what;
    running->wait_on = on;
    emu_yield();
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
    ++emu_progress;
    bar_release_if_complete();
    while (bar_generation == gen) emu_wait_yield("__syncthreads", nullptr);
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
struct CpCopy { void* dst; const void* src; size_t bytes, src_bytes; size_t group; };       // src_bytes < bytes: the rest is zero-filled
void cp_land(void* dst, const void* src, size_t bytes, size_t src_bytes) {
    if (src_bytes) std::memcpy(dst, src, src_bytes);
    std::memset((unsigned char*)dst + src_bytes, 0, bytes - src_bytes);
}
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

void emu_cp_async_zfill(void* dst, const void* src, size_t bytes, size_t src_bytes) {
    if (!cp_late()) { cp_land(dst, src, bytes, src_bytes); return; }
    CpQueue& q = cp_queue();
    q.copies.push_back({dst, src, bytes, src_bytes, q.committed});
}

void emu_cp_async(void* dst, const void* src, size_t bytes) { emu_cp_async_zfill(dst, src, bytes, bytes); }

void emu_cp_commit() { ++cp_queue().committed; }

void emu_cp_wait(int n) {
    CpQueue& q = cp_queue();
    if (q.committed <= (size_t)n) return;
    const size_t retire = q.committed - (size_t)n;        // groups 0 .. retire - 1 complete
    while (q.head < q.copies.size() && q.copies[q.head].group < retire) {
        const CpCopy& c = q.copies[q.head++];
        cp_land(c.dst, c.src, c.bytes, c.src_bytes);
    }
    if (q.head == q.copies.size()) { q.copies.clear(); q.head = 0; }
}

// static shared arrays poisoned so far by the running block
static thread_local std::vector<void*> static_smem_seen;
void emu_static_smem(void* p, size_t bytes) {
    for (void* q : static_smem_seen) if (q == p) return;
    static_smem_seen.push_back(p);
    std::memset(p, 0xA5, bytes);
}

// mbarriers and bulk copies.  Copies queued under DB_EMU_BULK=late, in issue order; a wait on a barrier lands that barrier's copies.
namespace {
struct BulkCopy { unsigned long long* bar; void* dst; const void* src; unsigned bytes; };
thread_local std::vector<BulkCopy> bulk_queue;
bool bulk_late() {
    static const bool late = [] {
        const char* e = getenv("DB_EMU_BULK");
        if (!e || !strcmp(e, "late")) return true;
        if (!strcmp(e, "early")) return false;
        fprintf(stderr, "DB_EMU_BULK=%s: expected 'late' or 'early'\n", e);
        abort();
    }();
    return late;
}
[[noreturn]] void emu_fail(const char* fmt, ...) __attribute__((format(printf, 1, 2)));
void emu_fail(const char* fmt, ...) {
    const EmuState& s = emu_cur;
    fprintf(stderr, "emu: block (%u,%u,%u) thread (%u,%u,%u): ", s.bid.x, s.bid.y, s.bid.z, s.tid.x, s.tid.y, s.tid.z);
    va_list ap;
    va_start(ap, fmt);
    vfprintf(stderr, fmt, ap);
    va_end(ap);
    fputc('\n', stderr);
    abort();
}
void check_bar(const unsigned long long* bar, const char* what) {
    if ((uintptr_t)bar % 8) emu_fail("%s: mbarrier %p is not 8-byte aligned", what, (const void*)bar);
}
// one copy lands: its bytes complete on the barrier; the phase completes when none are left
void bulk_land(const BulkCopy& c) {
    std::memcpy(c.dst, c.src, c.bytes);
    const unsigned pending = (unsigned)(*c.bar & 0xffffffffull);
    if (c.bytes > pending)
        emu_fail("bulk copy of %u bytes completes on mbarrier %p, which expects only %u more bytes in this phase", c.bytes, (void*)c.bar, pending);
    *c.bar -= c.bytes;
    ++emu_progress;
    if (pending == c.bytes) {
        for (const BulkCopy& o : bulk_queue)
            if (o.bar == c.bar) emu_fail("mbarrier %p completed its phase with a %u-byte bulk copy still in flight", (void*)c.bar, o.bytes);
        *c.bar += 1ull << 32;
    }
}
}  // namespace

void emu_check_align16(const void* p, const char* what) {
    if ((uintptr_t)p % 16) emu_fail("%s: 16-byte access at %p, which is not 16-byte aligned", what, p);
}

void emu_mbar_init(unsigned long long* bar) {
    check_bar(bar, "mbarrier.init");
    *bar = 0;
    ++emu_progress;
}

void emu_mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
    check_bar(bar, "mbarrier.arrive.expect_tx");
    *bar += bytes;
    ++emu_progress;
}

void emu_bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
    check_bar(bar, "cp.async.bulk");
    if ((uintptr_t)dst % 16 || (uintptr_t)src % 16) emu_fail("cp.async.bulk: addresses %p <- %p are not 16-byte aligned", dst, src);
    if (bytes == 0 || bytes % 16) emu_fail("cp.async.bulk: size %u is not a non-zero multiple of 16", bytes);
    const BulkCopy c{bar, dst, src, bytes};
    if (bulk_late()) { bulk_queue.push_back(c); ++emu_progress; }
    else bulk_land(c);
}

void emu_mbar_wait(unsigned long long* bar, unsigned parity) {
    check_bar(bar, "mbarrier.try_wait");
    while (((*bar >> 32) & 1ull) == parity) {
        // land this barrier's queued copies, oldest first
        bool landed = false;
        for (size_t i = 0; i < bulk_queue.size();) {
            if (bulk_queue[i].bar != bar) { ++i; continue; }
            const BulkCopy c = bulk_queue[i];
            bulk_queue.erase(bulk_queue.begin() + i);
            bulk_land(c);
            landed = true;
        }
        if (!landed) emu_wait_yield("mbarrier", bar);
    }
}

// arrival-count barrier: bits 0-15 pending arrivals, bits 16-31 arrivals per phase, bits 32.. completed phases
void emu_cbar_init(unsigned long long* bar, int count) {
    check_bar(bar, "mbarrier.init");
    *bar = (unsigned long long)count | ((unsigned long long)count << 16);
    ++emu_progress;
}

void emu_cbar_arrive(unsigned long long* bar) {
    check_bar(bar, "mbarrier.arrive");
    if ((*bar & 0xffffull) == 0) emu_fail("mbarrier.arrive on %p: more arrivals than the barrier counts", (void*)bar);
    *bar -= 1;
    if ((*bar & 0xffffull) == 0) *bar += (1ull << 32) + ((*bar >> 16) & 0xffffull);
    ++emu_progress;
}

void emu_launch(dim3 grid, dim3 block, size_t smem, const char* name, const std::function<void()>& body) {
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
        bulk_queue.clear();
        static_smem_seen.clear();
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
            size_t finished_this_round = 0, waiting = 0, blocked = 0;
            const size_t progress0 = emu_progress;
            const Fiber* first_blocked = nullptr;
            for (size_t fi = 0; fi < nthreads; ++fi) {
                Fiber& f = fibers[reverse_order ? nthreads - 1 - fi : fi];
                if (f.done) continue;
                f.wait_what = nullptr;
                resume(f);
                if (f.done) { ++finished_this_round; --bar_live; bar_release_if_complete(); } else { ++waiting; }
                if (!f.done && f.wait_what) { ++blocked; if (!first_blocked) first_blocked = &f; }
            }
            if (!finished_this_round && blocked == waiting && emu_progress == progress0) {
                const EmuState& s = first_blocked->st;
                fprintf(stderr, "emu_launch: deadlock in %s: block (%u,%u,%u) has %zu live threads, all waiting, and a whole round changed "
                        "nothing; thread (%u,%u,%u) waits at %s %p\n", name, s.bid.x, s.bid.y, s.bid.z, waiting, s.tid.x, s.tid.y, s.tid.z,
                        first_blocked->wait_what, first_blocked->wait_on);
                abort();
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
