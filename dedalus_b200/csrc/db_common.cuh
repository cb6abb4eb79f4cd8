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
__device__ __forceinline__ void db_cp_commit() { emu_cp_commit(); }
template <int N> __device__ __forceinline__ void db_cp_wait() { emu_cp_wait(N); }
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
__device__ __forceinline__ void db_cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void db_cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
#endif

#include "../../include/dedalus_b200.h"

// error plumbing (thread-compatible: one stream per rank, last error per process)
void db_set_error(const char* fmt, ...);
int db_check_launch(const char* what);
// streaming multiprocessors of the current device (grid-size caps of the grid-stride kernels)
int db_num_sms();

#define DB_MAX_SMEM (227 * 1024)
