// Common definitions for the dedalus_b200 CUDA kernels (sm_90a).
#pragma once
#ifdef DB_EMU
#include "cuda_emu.h"
#else
#include <cuda_runtime.h>
#include <cstdio>
#include <cstring>
#include <cmath>
#define DB_LAUNCH(kern, grid, block, smem, stream, ...) \
    kern<<<(grid), (block), (smem), (cudaStream_t)(stream)>>>(__VA_ARGS__)
#define DB_SMEM(type, name) \
    extern __shared__ __align__(16) unsigned char db_smem_raw[]; \
    type* name = reinterpret_cast<type*>(db_smem_raw)
#define DB_SET_SMEM_ATTR(kern) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024)
#endif

// a 16-byte global access (double2) must be 16-byte aligned: the emulation checks the address and aborts with a message, the GPU
// build compiles nothing
#ifdef DB_EMU
#define DB_CHECK_ALIGN16(p) emu_check_align16((const void*)(p), __func__)
#else
#define DB_CHECK_ALIGN16(p) ((void)0)
#endif

#ifdef DB_EMU
#define DB_LDCS(p) (*(p))
#else
#define DB_LDCS(p) __ldcs(p)           // streaming (evict-first) load: one-pass data must not displace reused lines
#endif

// asynchronous global -> shared copies (LDGSTS) used for deep software prefetch without register cost
#ifdef DB_EMU
// (the emulation defers each copy until a wait retires its group: tests/emu/cuda_emu.h)
__device__ __forceinline__ void db_cp_async8(void* dst, const void* src) { emu_cp_async(dst, src, 8); }
__device__ __forceinline__ void db_cp_async4(void* dst, const void* src) { emu_cp_async(dst, src, 4); }
__device__ __forceinline__ void db_cp_async16(void* dst, const void* src) { emu_cp_async(dst, src, 16); }
// 16 bytes, or 16 bytes of zeros when !valid (src is then not read)
__device__ __forceinline__ void db_cp_async16_zfill(void* dst, const void* src, bool valid) { emu_cp_async_zfill(dst, src, 16, valid ? 16 : 0); }
__device__ __forceinline__ void db_cp_commit() { emu_cp_commit(); }
template <int N> __device__ __forceinline__ void db_cp_wait() { emu_cp_wait(N); }
// the warp-wide 8 x 8 x 4 product C += A B from its fragments: lane t holds A[t/4][t%4], B[t%4][t/4] and C[t/4][2 (t%4) + {0, 1}],
// so it fetches row t/4 of A from lanes 4 (t/4) + k and columns 2 (t%4), 2 (t%4) + 1 of B from lanes 4 j + k
__device__ __forceinline__ void db_dmma_m8n8k4(double& c0, double& c1, double a, double b)
{
    const int lane = (int)(threadIdx.x & 31), i = lane >> 2, j = 2 * (lane & 3);
    for (int k = 0; k < 4; ++k) {
        const double ak = emu_shfl_exchange(a, 4 * i + k);
        const double b0 = emu_shfl_exchange(b, 4 * j + k), b1 = emu_shfl_exchange(b, 4 * (j + 1) + k);
        c0 = fma(ak, b0, c0); c1 = fma(ak, b1, c1);
    }
}
#else
__device__ __forceinline__ void db_cp_async8(void* dst, const void* src)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void db_cp_async4(void* dst, const void* src)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void db_cp_async16(void* dst, const void* src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
// 16 bytes, or 16 bytes of zeros when !valid (src-size 0: src is not read, but must be a valid address)
__device__ __forceinline__ void db_cp_async16_zfill(void* dst, const void* src, bool valid)
{
    const unsigned sz = valid ? 16u : 0u;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void db_cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void db_cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
// FP64 tensor-core product C += A B (8 x 8 x 4, DMMA): lane t holds A[t/4][t%4], B[t%4][t/4] and C[t/4][2 (t%4) + {0, 1}]
__device__ __forceinline__ void db_dmma_m8n8k4(double& c0, double& c1, double a, double b)
{
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
#endif

// a statically sized shared-memory array (the emulation keeps one host array per kernel and poisons it for every block)
#ifdef DB_EMU
#define DB_SHARED_ARRAY(type, name, dims) static type name dims; emu_static_smem(name, sizeof(name))
#else
#define DB_SHARED_ARRAY(type, name, dims) __shared__ __align__(16) type name dims
#endif

#include "../../include/dedalus_b200.h"

// error plumbing (thread-compatible: one stream per rank, last error per process)
void db_set_error(const char* fmt, ...);
int db_check_launch(const char* what);
// streaming multiprocessors of the current device (grid-size caps of the grid-stride kernels)
int db_num_sms();

#define DB_MAX_SMEM (227 * 1024)
