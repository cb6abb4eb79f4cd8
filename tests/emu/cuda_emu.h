// TEST INFRASTRUCTURE ONLY -- never linked into the product library.
// Minimal single-process emulation of the CUDA execution model so that the kernels in
// dedalus_b200/csrc/*.cu can be compiled with g++ (-x c++ -DDB_EMU) and their indexing / barrier logic
// checked on the GPU-less build container.  One CUDA thread = one ucontext fiber; __syncthreads() yields to
// a round-robin block scheduler.  Blocks run one after another.  The emulated library is built as
// tests/emu/libdedalus_b200_emu.so and loaded only by tests (tests/emu/emu_lib.py).
#pragma once
#include <ucontext.h>
#include <csetjmp>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include <functional>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)
#define __noinline__
#define __align__(x)

struct uint3e { unsigned x, y, z; };
struct dim3 {
    unsigned x, y, z;
    dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct double2 { double x, y; };
struct int4 { int x, y, z, w; };
static inline double2 make_double2(double x, double y) { double2 r; r.x = x; r.y = y; return r; }
typedef void* cudaStream_t;
typedef int cudaError_t;
#define cudaSuccess 0
static inline cudaError_t cudaGetLastError() { return 0; }
static inline const char* cudaGetErrorString(cudaError_t) { return "emu"; }

struct EmuState {
    uint3e tid, bid; dim3 bdim, gdim;
    unsigned char* smem;
};
extern thread_local EmuState emu_cur;           // state of the running fiber
#define threadIdx (emu_cur.tid)
#define blockIdx (emu_cur.bid)
#define blockDim (emu_cur.bdim)
#define gridDim (emu_cur.gdim)

void emu_syncthreads();
void emu_yield();          // one scheduling step (used by the emulated mbarrier wait and warp shuffles)
#define __syncthreads() emu_syncthreads()
#define __syncwarp(...) ((void)0)
// warp shuffles: every lane of the warp publishes its value, yields once (all live fibers advance one step per
// scheduler round), reads the source lane's slot, and yields again before any slot can be overwritten
double emu_shfl_exchange(double v, int src_lane);
static inline double __shfl_sync(unsigned, double v, int src) { return emu_shfl_exchange(v, src & 31); }
static inline double __shfl_down_sync(unsigned, double v, int off)
{
    const int lane = (int)(emu_cur.tid.x & 31);
    return emu_shfl_exchange(v, lane + off < 32 ? lane + off : lane);
}
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline void sincospi(double x, double* s, double* c) { *s = sin(M_PI * x); *c = cos(M_PI * x); }
static inline double atomicAdd(double* p, double v) { double o = *p; *p += v; return o; }
static inline int atomicAdd(int* p, int v) { int o = *p; *p += v; return o; }
static inline int atomicMax(int* p, int v) { int o = *p; if (v > o) *p = v; return o; }
static inline int atomicOr(int* p, int v) { int o = *p; *p |= v; return o; }

// asynchronous global -> shared copies (cp.async): each thread keeps its own queue of committed groups.  With DB_EMU_CP=late (the
// default) a copy lands only when a wait retires its group, so shared memory read before that still holds the 0xA5 poison (or an
// older value); with DB_EMU_CP=early it lands at issue, so a slot refilled while other code still reads it shows the new value.
void emu_cp_async(void* dst, const void* src, size_t bytes);
// the zero-filling form (cp.async ..., cp-size, src-size): src_bytes <= bytes are copied and the rest of dst is set to zero, when the
// copy lands; with src_bytes == 0 the source is not read at all
void emu_cp_async_zfill(void* dst, const void* src, size_t bytes, size_t src_bytes);
void emu_cp_commit();                // close the open group (also when it is empty), as cp.async.commit_group
void emu_cp_wait(int n);             // land every committed group except the n most recent, as cp.async.wait_group n

// a 16-byte global load or store (double2) at p, in kernel `what`: aborts with a message unless p is 16-byte aligned (the GPU faults
// with a misaligned address there, while host memory would take it silently)
void emu_check_align16(const void* p, const char* what);

// a statically sized __shared__ array (DB_SHARED_ARRAY): one host array shared by the fibers; the first thread of every block to reach
// the declaration poisons it, as emu_launch poisons the dynamic shared memory
void emu_static_smem(void* p, size_t bytes);

// mbarriers and 1-D bulk copies (cp.async.bulk ... mbarrier::complete_tx::bytes).  A barrier is one 64-bit word: low 32 bits = bytes
// still expected in the current phase (or, for an arrival-count barrier, pending arrivals and arrivals per phase), high 32 bits =
// completed phases.  With DB_EMU_BULK=late (the default) a bulk copy is queued on its barrier and lands, in issue order, only when a
// thread waits on that barrier: a stage read before its wait still holds the poison.  With DB_EMU_BULK=early it lands at issue.
// Either way the PTX rules are enforced (16-byte aligned addresses, a size that is a non-zero multiple of 16, an 8-byte aligned
// barrier, exactly the expect_tx bytes per phase), and a violation aborts with a message.
void emu_mbar_init(unsigned long long* bar);
void emu_mbar_expect_tx(unsigned long long* bar, unsigned bytes);
void emu_bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar);
void emu_mbar_wait(unsigned long long* bar, unsigned parity);
void emu_cbar_init(unsigned long long* bar, int count);
void emu_cbar_arrive(unsigned long long* bar);

// A launch aborts, naming the block and a waiting thread, when a whole scheduling round passes in which every live thread is
// blocked in an emulated wait (__syncthreads, mbarrier) and no barrier or copy-queue state changes: on the GPU it would hang.
void emu_launch(dim3 grid, dim3 block, size_t smem, const char* name, const std::function<void()>& body);

#define DB_LAUNCH(kern, grid, block, smem, stream, ...) \
    emu_launch(dim3(grid), dim3(block), (size_t)(smem), #kern, [&]() { kern(__VA_ARGS__); })
#define DB_SMEM(type, name) type* name = reinterpret_cast<type*>(emu_cur.smem)
#define DB_SET_SMEM_ATTR(kern) ((void)0)
