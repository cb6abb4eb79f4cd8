// Batched pencil-system kernels, structure-of-arrays, one thread per system.
//
// Reference behaviour replaced: the per-pencil Python loops of core/timesteppers.py:588-643 (gather, CSR
// mat-vecs, RHS axpy, SuperLU solve, scatter) and core/subsystems.py:340-371.
// Design: every batch is S structurally identical systems; thread s owns system s, arrays are
// [row or entry][system] so a warp's 32 loads of one entry are one 256-byte coalesced transaction and the
// integer program (shared by all systems) is read uniformly.  The LU values are stored in the exact order
// the triangular solves consume them, so the solve is a pure stream over the factors.
#include "db_common.cuh"
#include <cstdlib>

#define PB_THREADS 128

// Tile-major storage of every [rows][systems] array of a batch (vectors: rows = n, factors: rows = n_entries):
//   element (i, s)  ->  ((s / DB_TILE) * rows + i) * DB_TILE + (s % DB_TILE)
// Each group of DB_TILE = 64 systems (one solve CTA) owns ONE contiguous slab that it streams front to back, so the
// dominant factor stream is sequential in DRAM (row-buffer and TLB friendly) instead of striding by the batch size.
__device__ __forceinline__ int64_t db_tbase(int s, int rows) { return ((int64_t)(s / DB_TILE) * rows) * DB_TILE + (s % DB_TILE); }

// ---------------------------------------------------------------------------------------------------------
// gather / scatter: tiled transposes between z-contiguous field lines and system-contiguous pencil vectors
// ---------------------------------------------------------------------------------------------------------
template <bool GATHER>
__global__ void k_pencil_move(const double* __restrict__ src, double* __restrict__ dst, int S, int nrows,
                              const int64_t* __restrict__ line_base, const int32_t* __restrict__ line_kind,
                              const int32_t* __restrict__ line_ptr, const int32_t* __restrict__ line_pos,
                              const int64_t* __restrict__ sys_off, int ld_sys)
{
    // block (32, 8): tile of 32 modes x 32 systems of line blockIdx.z
    DB_SMEM(double, tile);                      // [32][33]
    const int q = blockIdx.z;
    const int len = line_ptr[q + 1] - line_ptr[q];
    const int m0 = blockIdx.y * 32;
    if (m0 >= len) return;
    const int s0 = blockIdx.x * 32;
    const int64_t base = line_base[q];
    const int64_t* so = sys_off + (int64_t)line_kind[q] * ld_sys;
    const int32_t* pos = line_pos + line_ptr[q];
    const int tx = threadIdx.x, ty = threadIdx.y;
    if (GATHER) {
        for (int r = ty; r < 32; r += 8) {       // read arena: tx -> mode (contiguous)
            int s = s0 + r, m = m0 + tx;
            if (s < S && m < len) tile[r * 33 + tx] = src[base + so[s] + m];
        }
        __syncthreads();
        for (int r = ty; r < 32; r += 8) {       // write vec: tx -> system (contiguous)
            int m = m0 + r, s = s0 + tx;
            if (s < S && m < len) dst[db_tbase(s, nrows) + (int64_t)pos[m] * DB_TILE] = tile[tx * 33 + r];
        }
    } else {
        for (int r = ty; r < 32; r += 8) {
            int m = m0 + r, s = s0 + tx;
            if (s < S && m < len) tile[tx * 33 + r] = src[db_tbase(s, nrows) + (int64_t)pos[m] * DB_TILE];
        }
        __syncthreads();
        for (int r = ty; r < 32; r += 8) {
            int s = s0 + r, m = m0 + tx;
            if (s < S && m < len) dst[base + so[s] + m] = tile[r * 33 + tx];
        }
    }
}

extern "C" int db_pencil_gather(const double* arena, double* vec, int32_t S, int32_t n, int32_t nlines, int32_t max_len,
                                const int64_t* line_base, const int32_t* line_kind, const int32_t* line_ptr, const int32_t* line_pos,
                                const int64_t* sys_off, int32_t ld_sys, void* stream)
{
    if (S <= 0 || nlines <= 0 || max_len <= 0) return 0;
    dim3 grid((S + 31) / 32, (max_len + 31) / 32, nlines), block(32, 8);
    DB_LAUNCH(k_pencil_move<true>, grid, block, 32 * 33 * sizeof(double), stream, arena, vec, S, n, line_base, line_kind, line_ptr, line_pos, sys_off, ld_sys);
    return db_check_launch("pencil_gather");
}

extern "C" int db_pencil_scatter(const double* vec, double* arena, int32_t S, int32_t n, int32_t nlines, int32_t max_len,
                                 const int64_t* line_base, const int32_t* line_kind, const int32_t* line_ptr, const int32_t* line_pos,
                                 const int64_t* sys_off, int32_t ld_sys, void* stream)
{
    if (S <= 0 || nlines <= 0 || max_len <= 0) return 0;
    dim3 grid((S + 31) / 32, (max_len + 31) / 32, nlines), block(32, 8);
    DB_LAUNCH(k_pencil_move<false>, grid, block, 32 * 33 * sizeof(double), stream, vec, arena, S, n, line_base, line_kind, line_ptr, line_pos, sys_off, ld_sys);
    return db_check_launch("pencil_scatter");
}

// ---------------------------------------------------------------------------------------------------------
// template mat-vecs  y = (sum_mono mono_vals[mono][s] T_mono) x   for M and L in one pass over rows
// grid: (ceil(S/128), row chunks)
// ---------------------------------------------------------------------------------------------------------
#define MV_ROWS_PER_BLOCK 64
__global__ void k_pencil_matvec(int n, int S, int ld, const double* __restrict__ mono_vals, const double* x,
                                const int32_t* __restrict__ m_ptr, const int32_t* __restrict__ m_col, const int32_t* __restrict__ m_mono, const double* __restrict__ m_val, double* y_m,
                                const int32_t* __restrict__ l_ptr, const int32_t* __restrict__ l_col, const int32_t* __restrict__ l_mono, const double* __restrict__ l_val, double* y_l)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    const int r0 = blockIdx.y * MV_ROWS_PER_BLOCK;
    const int r1 = (r0 + MV_ROWS_PER_BLOCK < n) ? r0 + MV_ROWS_PER_BLOCK : n;
    const int64_t tb = db_tbase(s, n);
    x += tb; if (y_m) y_m += tb; if (y_l) y_l += tb;
    for (int i = r0; i < r1; ++i) {
        if (y_m) {
            double acc = 0.0;
            for (int t = m_ptr[i]; t < m_ptr[i + 1]; ++t)
                acc = fma(m_val[t] * mono_vals[(int64_t)m_mono[t] * ld + s], x[(int64_t)m_col[t] * DB_TILE], acc);
            y_m[(int64_t)i * DB_TILE] = acc;
        }
        if (y_l) {
            double acc = 0.0;
            for (int t = l_ptr[i]; t < l_ptr[i + 1]; ++t)
                acc = fma(l_val[t] * mono_vals[(int64_t)l_mono[t] * ld + s], x[(int64_t)l_col[t] * DB_TILE], acc);
            y_l[(int64_t)i * DB_TILE] = acc;
        }
    }
}

extern "C" int db_pencil_matvec(int32_t n, int32_t S, int32_t ld, const double* mono_vals, const double* x,
                                const int32_t* m_ptr, const int32_t* m_col, const int32_t* m_mono, const double* m_val, double* y_m,
                                const int32_t* l_ptr, const int32_t* l_col, const int32_t* l_mono, const double* l_val, double* y_l,
                                void* stream)
{
    if (S <= 0 || n <= 0) return 0;
    dim3 grid((S + PB_THREADS - 1) / PB_THREADS, (n + MV_ROWS_PER_BLOCK - 1) / MV_ROWS_PER_BLOCK), block(PB_THREADS);
    DB_LAUNCH(k_pencil_matvec, grid, block, 0, stream, n, S, ld, mono_vals, x, m_ptr, m_col, m_mono, m_val, y_m, l_ptr, l_col, l_mono, l_val, y_l);
    return db_check_launch("pencil_matvec");
}

// ---------------------------------------------------------------------------------------------------------
// LHS assembly on the static fill pattern
// ---------------------------------------------------------------------------------------------------------
#define ASM_ENTRIES_PER_BLOCK 64
__global__ void k_pencil_assemble(double* __restrict__ lu, int n_entries, int S, int ld, const double* __restrict__ mono_vals,
                                  const int32_t* __restrict__ asm_ptr, const int32_t* __restrict__ asm_mono, const double* __restrict__ asm_val)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    const int e0 = blockIdx.y * ASM_ENTRIES_PER_BLOCK;
    const int e1 = (e0 + ASM_ENTRIES_PER_BLOCK < n_entries) ? e0 + ASM_ENTRIES_PER_BLOCK : n_entries;
    for (int e = e0; e < e1; ++e) {
        double v = 0.0;
        for (int t = asm_ptr[e]; t < asm_ptr[e + 1]; ++t)
            v = fma(asm_val[t], mono_vals[(int64_t)asm_mono[t] * ld + s], v);
        lu[db_tbase(s, n_entries) + (int64_t)e * DB_TILE] = v;
    }
}

extern "C" int db_pencil_assemble(double* lu, int32_t n_entries, int32_t S, int32_t ld, const double* mono_vals,
                                  const int32_t* asm_ptr, const int32_t* asm_mono, const double* asm_val, void* stream)
{
    if (S <= 0 || n_entries <= 0) return 0;
    dim3 grid((S + PB_THREADS - 1) / PB_THREADS, (n_entries + ASM_ENTRIES_PER_BLOCK - 1) / ASM_ENTRIES_PER_BLOCK), block(PB_THREADS);
    DB_LAUNCH(k_pencil_assemble, grid, block, 0, stream, lu, n_entries, S, ld, mono_vals, asm_ptr, asm_mono, asm_val);
    return db_check_launch("pencil_assemble");
}

// ---------------------------------------------------------------------------------------------------------
// numeric LU on the static schedule (no pivot search: the order was fixed by the host's joint threshold
// pivoting); reciprocal pivots are stored on the diagonal
// ---------------------------------------------------------------------------------------------------------
__global__ void k_pencil_factor(double* __restrict__ lu, int n, int S, int n_entries, const int32_t* __restrict__ diag_eid,
                                const int32_t* __restrict__ fl_ptr, const int32_t* __restrict__ fl_eid,
                                const int32_t* __restrict__ fu_ptr, const int32_t* __restrict__ fu_eid,
                                const int32_t* __restrict__ fd_eid, int32_t* __restrict__ info)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    int64_t dp = 0;
    bool bad = false;
    lu += db_tbase(s, n_entries);
    for (int k = 0; k < n; ++k) {
        const int64_t d = (int64_t)diag_eid[k] * DB_TILE;
        const double piv = lu[d];
        if (!(fabs(piv) > 0.0) || !(fabs(piv) < 1e300)) bad = true;
        const double inv = 1.0 / piv;
        lu[d] = inv;
        const int u0 = fu_ptr[k], u1 = fu_ptr[k + 1];
        for (int a = fl_ptr[k]; a < fl_ptr[k + 1]; ++a) {
            const int64_t le = (int64_t)fl_eid[a] * DB_TILE;
            const double l = lu[le] * inv;
            lu[le] = l;
            for (int b = u0; b < u1; ++b, ++dp) {
                const int64_t de = (int64_t)fd_eid[dp] * DB_TILE;
                lu[de] = fma(-l, lu[(int64_t)fu_eid[b] * DB_TILE], lu[de]);
            }
        }
    }
    if (bad) atomicAdd(info, 1);
}

extern "C" int db_pencil_factor(double* lu, int32_t n, int32_t S, int32_t n_entries, const int32_t* diag_eid,
                                const int32_t* fl_ptr, const int32_t* fl_eid, const int32_t* fu_ptr, const int32_t* fu_eid,
                                const int32_t* fd_eid, int32_t* info, void* stream)
{
    if (S <= 0 || n <= 0) return 0;
    dim3 grid((S + 63) / 64), block(64);
    DB_LAUNCH(k_pencil_factor, grid, block, 0, stream, lu, n, S, n_entries, diag_eid, fl_ptr, fl_eid, fu_ptr, fu_eid, fd_eid, info);
    return db_check_launch("pencil_factor");
}

// ---------------------------------------------------------------------------------------------------------
// triangular solves streaming the factors (single batch; the fused multi-batch version is below)
// ---------------------------------------------------------------------------------------------------------
__global__ void k_pencil_solve(const double* __restrict__ lu, int n, int S, int ld,
                               const int32_t* __restrict__ prog, int n_fwd, int n_entries,
                               db_lincomb rhs, double* xg)
{
    // plain sequential interpreter of the solve stream (reference implementation; the fused branch-free kernel below
    // must agree with it): x <- right-hand-side combination, then every row starts from x[row]
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    (void)ld;
    const double* __restrict__ f = lu + db_tbase(s, n_entries);
    const int64_t tb = db_tbase(s, n);
    double* x = xg + tb;
    for (int i = 0; i < n; ++i) {
        double acc = 0.0;
        for (int j = 0; j < rhs.nvec; ++j) acc = fma(rhs.coef[j], rhs.vec[j][tb + (int64_t)i * DB_TILE], acc);
        x[(int64_t)i * DB_TILE] = acc;
    }
    for (int sec = 0; sec < 2; ++sec) {
        const int e0 = sec ? n_fwd : 0, e1 = sec ? n_entries : n_fwd;
        int cur = -1;
        double acc = 0.0;
        for (int e = e0; e < e1; ++e) {
            const int c = prog[e];
            if (c == DB_I_SKIP) continue;
            if (c < 0) {
                if (cur >= 0) x[cur] = sec ? acc * f[(int64_t)e * DB_TILE] : acc;
                cur = -1 - c;
                acc = x[cur];
            } else {
                acc = fma(-f[(int64_t)e * DB_TILE], x[c], acc);
            }
        }
    }
}

extern "C" int db_pencil_solve(const double* lu, int32_t n, int32_t S, int32_t ld,
                               const int32_t* prog, int32_t n_fwd, int32_t n_entries,
                               const db_lincomb* rhs, double* x, void* stream)
{
    if (S <= 0 || n <= 0) return 0;
    if (rhs->nvec < 0 || rhs->nvec > 16) { db_set_error("pencil_solve: nvec out of range"); return 1; }
    dim3 grid((S + 63) / 64), block(64);
    DB_LAUNCH(k_pencil_solve, grid, block, 0, stream, lu, n, S, ld, prog, n_fwd, n_entries, *rhs, x);
    return db_check_launch("pencil_solve");
}

// ---------------------------------------------------------------------------------------------------------
__global__ void k_lincomb(db_lincomb terms, double* __restrict__ out, int64_t count)
{
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) {
        double acc = 0.0;
        for (int j = 0; j < terms.nvec; ++j) acc = fma(terms.coef[j], terms.vec[j][i], acc);
        out[i] = acc;
    }
}

extern "C" int db_lincomb_apply(const db_lincomb* terms, double* out, int64_t count, void* stream)
{
    if (count <= 0) return 0;
    int64_t blocks = (count + 255) / 256;
    if (blocks > (int64_t)db_num_sms() * 16) blocks = (int64_t)db_num_sms() * 16;
    DB_LAUNCH(k_lincomb, dim3((unsigned)blocks), dim3(256), 0, stream, *terms, out, count);
    return db_check_launch("lincomb");
}

// =========================================================================================================
// Fused launches over all batches of a solver
// =========================================================================================================
__device__ __forceinline__ int find_batch(const db_batch* __restrict__ b, int nbatch, int blk, int which)
{
    // which: 0 solve, 1 matvec, 2 move side 0, 3 move side 1, 4 assemble.  Uniform linear scan (nbatch is small).
    int lo = 0;
    for (int i = 1; i < nbatch; ++i) {
        int start = (which == 0) ? b[i].blk_solve : (which == 1) ? b[i].blk_matvec : (which == 2) ? b[i].blk_move[0]
                  : (which == 3) ? b[i].blk_move[1] : b[i].blk_assemble;
        if (blk >= start) lo = i;
    }
    return lo;
}

#define SOLVE_THREADS 64              // lanes per member group = systems per tile
#define SOLVE_MAX_RHS 4               // members (right-hand sides per factorisation) one CTA can carry
// Right-hand side first: x <- sum_q cf[q] * rv[q] for every row, as one fully parallel streaming pass (many
// independent loads in flight per thread).  The forward sweep then starts each row from x[row] like the backward sweep
// does; folding the combination into the row starts instead puts NV dependent DRAM loads on the recurrence's critical
// path two or three times per 16-entry chunk (rows are short), which is what the sweep's time was made of.
#define SOLVE_PRO_U 8      /* rows per iteration: NV * 8 independent streaming loads in flight per thread (the prologue was 18 % of the
                              solve's stall samples at 4 rows: it is a pure DRAM stream, bound by loads in flight) */
#define SOLVE_PROLOGUE(NV_, NROWS)                                                                  \
    {                                                                                               \
        const int nrows_ = (NROWS);                                                                 \
        int i_ = 0;                                                                                 \
        for (; i_ + SOLVE_PRO_U <= nrows_; i_ += SOLVE_PRO_U) {                                     \
            double a_[SOLVE_PRO_U];                                                                 \
            _Pragma("unroll") for (int u_ = 0; u_ < SOLVE_PRO_U; ++u_) a_[u_] = 0.0;                \
            _Pragma("unroll") for (int q_ = 0; q_ < NV_; ++q_) {                                    \
                _Pragma("unroll") for (int u_ = 0; u_ < SOLVE_PRO_U; ++u_)                          \
                    a_[u_] = fma(cf[q_], DB_LDCS(rv[q_] + (int64_t)(i_ + u_) * DB_TILE), a_[u_]);   \
            }                                                                                       \
            _Pragma("unroll") for (int u_ = 0; u_ < SOLVE_PRO_U; ++u_) x[(int64_t)(i_ + u_) * DB_TILE] = a_[u_]; \
        }                                                                                           \
        for (; i_ < nrows_; ++i_) {                                                                 \
            double a_ = 0.0;                                                                        \
            _Pragma("unroll") for (int q_ = 0; q_ < NV_; ++q_) a_ = fma(cf[q_], DB_LDCS(rv[q_] + (int64_t)i_ * DB_TILE), a_); \
            x[(int64_t)i_ * DB_TILE] = a_;                                                          \
        }                                                                                           \
    }

// ---------------------------------------------------------------------------------------------------------
// Bulk-copy ring.  The tile-major factor array makes everything one CTA (64 systems) reads a single contiguous stream
// of n_entries * 512 bytes, so one elected thread feeds it through a ring of shared-memory stages with 1-D bulk async
// copies (cp.async.bulk -> UBLKCP) completing on mbarriers; the control block of each chunk rides in the same stage.
// The copy engine keeps `nstages` chunks in flight per CTA no matter how few warps are resident, which is what a
// one-thread-per-system recurrence needs when there are only a few tiles per SM (multi-GPU strong scaling).
// ---------------------------------------------------------------------------------------------------------
#define SOLVE_CE 16
#ifdef DB_EMU
// test emulation (tests/emu/cuda_emu.h): bulk copies are queued on their mbarrier and land when a thread waits on it
// (DB_EMU_BULK=late) or at issue (early); a waiter yields to the other fibers until the phase it waits for is complete
typedef unsigned long long db_mbar_t;
__device__ __forceinline__ void db_mbar_init(db_mbar_t* bar, int) { emu_mbar_init(bar); }
__device__ __forceinline__ void db_mbar_fence_init() {}
__device__ __forceinline__ void db_mbar_expect_tx(db_mbar_t* bar, unsigned bytes) { emu_mbar_expect_tx(bar, bytes); }
__device__ __forceinline__ void db_bulk_g2s(void* dst, const void* src, unsigned bytes, db_mbar_t* bar) { emu_bulk_g2s(dst, src, bytes, bar); }
__device__ __forceinline__ void db_mbar_wait(db_mbar_t* bar, unsigned parity) { emu_mbar_wait(bar, parity); }
__device__ __forceinline__ void db_cbar_init(db_mbar_t* bar, int count) { emu_cbar_init(bar, count); }
__device__ __forceinline__ void db_cbar_arrive(db_mbar_t* bar) { emu_cbar_arrive(bar); }
#define DB_CBAR_PER_THREAD 1        // every consumer thread arrives (fibers are not warp-synchronous)
#else
typedef unsigned long long db_mbar_t;
__device__ __forceinline__ unsigned db_smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void db_mbar_init(db_mbar_t* bar, int count)
{ asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(db_smem_u32(bar)), "r"(count) : "memory"); }
__device__ __forceinline__ void db_mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void db_mbar_expect_tx(db_mbar_t* bar, unsigned bytes)
{ asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(db_smem_u32(bar)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void db_bulk_g2s(void* dst, const void* src, unsigned bytes, db_mbar_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(db_smem_u32(dst)), "l"(src), "r"(bytes), "r"(db_smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void db_cbar_init(db_mbar_t* bar, int count) { db_mbar_init(bar, count); }
__device__ __forceinline__ void db_cbar_arrive(db_mbar_t* bar)
{ asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(db_smem_u32(bar)) : "memory"); }
#define DB_CBAR_PER_THREAD 0        // one elected lane per consumer warp arrives after __syncwarp()
__device__ __forceinline__ void db_mbar_wait(db_mbar_t* bar, unsigned parity)
{
    asm volatile("{\n"
                 ".reg .pred P1;\n"
                 "LAB_WAIT:\n"
                 "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
                 "@P1 bra DONE;\n"
                 "bra LAB_WAIT;\n"
                 "DONE:\n"
                 "}" ::"r"(db_smem_u32(bar)), "r"(parity) : "memory");
}
#endif


// ---------------------------------------------------------------------------------------------------------
// Triangular solves, branch-free variant on the same bulk-copy ring.  The interpreter above decodes one instruction
// word per entry (load -> compare -> branch), which with one or two warps per scheduler costs ~200 cycles per entry
// and is what kept the sweep from scaling to fewer systems per GPU.  Here the host pre-decodes each 16-entry chunk
// into a control block (gather offsets, finished-row offsets, three 16-bit masks; dedalus_b200/pencils.py
// solve_control_blocks) and the chunk is straight-line code: 16 gathers, then per entry one shared-memory load, one
// FMA, a predicated store and a select; chunks made only of multiply-accumulates (the dense boundary rows: a third of
// all entries) take a shorter path.
// ---------------------------------------------------------------------------------------------------------
#define SOLVE_CTRL_WORDS 44
// Start values of the rows entered SOLVE_PF_AHEAD chunks from now (control words 41, 42): pulled towards the SM early, so
// that the gather at the row's first entry hits a cache instead of paying a DRAM round trip on the thread's critical path
#ifdef DB_EMU
#define DB_PREFETCH_L2(p) ((void)0)
#define DB_PREFETCH_L1(p) ((void)0)
#else
#define DB_PREFETCH_L2(p) asm volatile("prefetch.global.L2 [%0];" ::"l"(p))
#define DB_PREFETCH_L1(p) asm volatile("prefetch.global.L1 [%0];" ::"l"(p))
#endif
__device__ __forceinline__ void solve_prefetch(const int* __restrict__ ctrl, const double* x, int mode)
{
    if (mode == 0) return;
    const int p0 = ctrl[41], p1 = ctrl[42];
    if (mode == 1) { if (p0 >= 0) DB_PREFETCH_L2(x + p0); if (p1 >= 0) DB_PREFETCH_L2(x + p1); }
    else { if (p0 >= 0) DB_PREFETCH_L1(x + p0); if (p1 >= 0) DB_PREFETCH_L1(x + p1); }
}
#define SOLVE_FSTAGE_BYTES (SOLVE_CE * DB_TILE * 8 + SOLVE_CTRL_WORDS * 4)

template <bool FWD, bool LATE>
__device__ __forceinline__ double solve_chunk_flat(const double* __restrict__ vals, const int* __restrict__ ctrl, double* x, double acc)
{
    // register diet: the gather offsets are consumed straight from the control block and the finished-row / late offsets are
    // re-read from shared memory at the few entries that need them, so that only the 16 gathered values stay live.
    // (Also holding the 16 factor values in registers -- to take their shared-memory loads off the dependent chain --
    // costs more in occupancy / spills than it gains.)
    double xv[SOLVE_CE];
#pragma unroll
    for (int j = 0; j < SOLVE_CE; j += 4) {
        const int4 g = *reinterpret_cast<const int4*>(ctrl + j);
        xv[j] = x[g.x]; xv[j + 1] = x[g.y]; xv[j + 2] = x[g.z]; xv[j + 3] = x[g.w];
    }
    const unsigned maskE = (unsigned)ctrl[2 * SOLVE_CE], maskB = (unsigned)ctrl[2 * SOLVE_CE + 1], maskF = (unsigned)ctrl[2 * SOLVE_CE + 2];
#pragma unroll
    for (int j = 0; j < SOLVE_CE; ++j) {
        const double v = vals[j * DB_TILE];
        if (LATE) { if (maskF & (1u << j)) xv[j] = x[ctrl[j]]; }
        const double acc_a = fma(-v, xv[j], acc);
        const double val = FWD ? acc : acc * v;
        if (maskE & (1u << j)) x[ctrl[SOLVE_CE + j]] = val;
        acc = (maskB & (1u << j)) ? xv[j] : acc_a;
    }
    return acc;
}

__device__ __forceinline__ double solve_chunk_pure(const double* __restrict__ vals, const int* __restrict__ ctrl, const double* x, double acc)
{
    double xv[SOLVE_CE];
#pragma unroll
    for (int j = 0; j < SOLVE_CE; j += 4) {
        const int4 g = *reinterpret_cast<const int4*>(ctrl + j);
        xv[j] = x[g.x]; xv[j + 1] = x[g.y]; xv[j + 2] = x[g.z]; xv[j + 3] = x[g.w];
    }
#pragma unroll
    for (int j = 0; j < SOLVE_CE; ++j) acc = fma(-vals[j * DB_TILE], xv[j], acc);
    return acc;
}

template <int NV, int MINB>
__global__ void __launch_bounds__(SOLVE_THREADS * SOLVE_MAX_RHS, MINB)
k_batches_solve_flat(const db_batch* __restrict__ batches, int nbatch, int lu_slot, int x_slot, db_slotcomb rhs, int nstages_pf)
{
    const int nstages = nstages_pf & 255, pfmode = nstages_pf >> 8;       // ring depth | row-start prefetch mode << 8
    // blockDim.x = 64 * (largest nrhs of the launch).  Thread group g = threadIdx.x / 64 owns member g of the tile's 64
    // pencils: all groups consume the SAME factor stage of the ring (one DRAM read of the factors for nrhs solves); groups
    // beyond the batch's nrhs only take part in the barriers.
    DB_SMEM(unsigned char, ring);
    db_mbar_t* bars = reinterpret_cast<db_mbar_t*>(ring + (size_t)nstages * SOLVE_FSTAGE_BYTES);
    const int bi = find_batch(batches, nbatch, blockIdx.x, 0);
    const db_batch& B = batches[bi];
    const int tile = blockIdx.x - B.blk_solve;
    const int grp = threadIdx.x / SOLVE_THREADS, lane = threadIdx.x % SOLVE_THREADS;
    const bool active = grp < B.nrhs;
    const int s = (active ? grp : 0) * B.ld + tile * SOLVE_THREADS + lane;   // padded lanes run on the zero padding
    const int64_t tb = db_tbase(s, B.n);
    const double* __restrict__ lu_tile = B.lu[lu_slot] + (int64_t)tile * B.n_entries * DB_TILE;
    const int32_t* __restrict__ ctrl_g = B.ctrl;
    const int nchunks = B.n_entries / SOLVE_CE, nfwd = B.n_fwd / SOLVE_CE;
    double* x = B.vec[x_slot] + tb;
    const double* rv[NV];
    double cf[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) { rv[j] = B.vec[rhs.slot[j < rhs.nvec ? j : 0]] + tb; cf[j] = (j < rhs.nvec) ? rhs.coef[j] : 0.0; }
    auto issue = [&](int q, int slot) {
        unsigned char* st = ring + (size_t)slot * SOLVE_FSTAGE_BYTES;
        db_mbar_expect_tx(&bars[slot], SOLVE_FSTAGE_BYTES);
        db_bulk_g2s(st, lu_tile + (int64_t)q * SOLVE_CE * DB_TILE, SOLVE_CE * DB_TILE * 8, &bars[slot]);
        db_bulk_g2s(st + SOLVE_CE * DB_TILE * 8, ctrl_g + (int64_t)q * SOLVE_CTRL_WORDS, SOLVE_CTRL_WORDS * 4, &bars[slot]);
    };
    if (threadIdx.x == 0) {
        for (int i = 0; i < nstages; ++i) db_mbar_init(&bars[i], 1);
        db_mbar_fence_init();
    }
    __syncthreads();
    if (threadIdx.x == 0)
        for (int q = 0; q < nstages && q < nchunks; ++q) issue(q, q);
    if (active) SOLVE_PROLOGUE(NV, B.n)
    int slot = 0;
    unsigned phase = 0;
    double acc = 0.0;
    for (int q = 0; q < nchunks; ++q) {
        if (active) {
            db_mbar_wait(&bars[slot], phase);
            const unsigned char* st = ring + (size_t)slot * SOLVE_FSTAGE_BYTES;
            const double* __restrict__ vals = reinterpret_cast<const double*>(st) + lane;
            const int* __restrict__ ctrl = reinterpret_cast<const int*>(st + SOLVE_CE * DB_TILE * 8);
            const unsigned mB = (unsigned)ctrl[2 * SOLVE_CE + 1], mF = (unsigned)ctrl[2 * SOLVE_CE + 2];
            solve_prefetch(ctrl, x, pfmode);
            if ((mB | mF) == 0) acc = solve_chunk_pure(vals, ctrl, x, acc);
            else if (q < nfwd) acc = mF ? solve_chunk_flat<true, true>(vals, ctrl, x, acc) : solve_chunk_flat<true, false>(vals, ctrl, x, acc);
            else acc = mF ? solve_chunk_flat<false, true>(vals, ctrl, x, acc) : solve_chunk_flat<false, false>(vals, ctrl, x, acc);
        }
        __syncthreads();                                   // every warp is done with this stage
        if (threadIdx.x == 0 && q + nstages < nchunks) issue(q + nstages, slot);
        if (++slot == nstages) { slot = 0; phase ^= 1; }
    }
}


// ---------------------------------------------------------------------------------------------------------
// Software-pipelined variant (opt-in, DB_SOLVE_PIPE=1; not yet measured): the 16 gathers of chunk q+1 are issued BEFORE
// chunk q is consumed, so a CTA that is alone on its SM (multi-GPU strong scaling: one or two tiles per SM) overlaps the
// L2 / DRAM latency of the gathers with the dependent FMA chain of the previous chunk.  The hazard window grows by one
// chunk: control word 35 (maskF2) marks the entries whose source row is stored in this or the previous chunk.
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void solve_gather(const int* __restrict__ ctrl, const double* x, double (&xv)[SOLVE_CE])
{
#pragma unroll
    for (int j = 0; j < SOLVE_CE; j += 4) {
        const int4 g = *reinterpret_cast<const int4*>(ctrl + j);
        xv[j] = x[g.x]; xv[j + 1] = x[g.y]; xv[j + 2] = x[g.z]; xv[j + 3] = x[g.w];
    }
}

template <bool FWD>
__device__ __forceinline__ double solve_chunk_pipe(const double* __restrict__ vals, const int* __restrict__ ctrl, double* x,
                                                   double (&xv)[SOLVE_CE], double acc)
{
    const unsigned maskE = (unsigned)ctrl[2 * SOLVE_CE], maskB = (unsigned)ctrl[2 * SOLVE_CE + 1], maskL = (unsigned)ctrl[2 * SOLVE_CE + 3];
    if ((maskB | maskL) == 0) {
#pragma unroll
        for (int j = 0; j < SOLVE_CE; ++j) acc = fma(-vals[j * DB_TILE], xv[j], acc);
        return acc;
    }
    int goff[SOLVE_CE], foff[SOLVE_CE];
#pragma unroll
    for (int j = 0; j < SOLVE_CE; j += 4) {
        const int4 g = *reinterpret_cast<const int4*>(ctrl + j);
        goff[j] = g.x; goff[j + 1] = g.y; goff[j + 2] = g.z; goff[j + 3] = g.w;
        const int4 f = *reinterpret_cast<const int4*>(ctrl + SOLVE_CE + j);
        foff[j] = f.x; foff[j + 1] = f.y; foff[j + 2] = f.z; foff[j + 3] = f.w;
    }
#pragma unroll
    for (int j = 0; j < SOLVE_CE; ++j) {
        const double v = vals[j * DB_TILE];
        if (maskL & (1u << j)) xv[j] = x[goff[j]];
        const double acc_a = fma(-v, xv[j], acc);
        const double val = FWD ? acc : acc * v;
        if (maskE & (1u << j)) x[foff[j]] = val;
        acc = (maskB & (1u << j)) ? xv[j] : acc_a;
    }
    return acc;
}

template <int NV>
__global__ void __launch_bounds__(SOLVE_THREADS * SOLVE_MAX_RHS)
k_batches_solve_pipe(const db_batch* __restrict__ batches, int nbatch, int lu_slot, int x_slot, db_slotcomb rhs, int nstages)
{
    // blockDim.x = 64 * (largest nrhs of the launch).  Thread group g = threadIdx.x / 64 owns member g of the tile's 64
    // pencils: all groups consume the SAME factor stage of the ring (one DRAM read of the factors for nrhs solves); groups
    // beyond the batch's nrhs only take part in the barriers.
    DB_SMEM(unsigned char, ring);
    db_mbar_t* bars = reinterpret_cast<db_mbar_t*>(ring + (size_t)nstages * SOLVE_FSTAGE_BYTES);
    const int bi = find_batch(batches, nbatch, blockIdx.x, 0);
    const db_batch& B = batches[bi];
    const int tile = blockIdx.x - B.blk_solve;
    const int grp = threadIdx.x / SOLVE_THREADS, lane = threadIdx.x % SOLVE_THREADS;
    const bool active = grp < B.nrhs;
    const int s = (active ? grp : 0) * B.ld + tile * SOLVE_THREADS + lane;
    const int64_t tb = db_tbase(s, B.n);
    const double* __restrict__ lu_tile = B.lu[lu_slot] + (int64_t)tile * B.n_entries * DB_TILE;
    const int32_t* __restrict__ ctrl_g = B.ctrl;
    const int nchunks = B.n_entries / SOLVE_CE, nfwd = B.n_fwd / SOLVE_CE;
    double* x = B.vec[x_slot] + tb;
    const double* rv[NV];
    double cf[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) { rv[j] = B.vec[rhs.slot[j < rhs.nvec ? j : 0]] + tb; cf[j] = (j < rhs.nvec) ? rhs.coef[j] : 0.0; }
    auto issue = [&](int q, int slot) {
        unsigned char* st = ring + (size_t)slot * SOLVE_FSTAGE_BYTES;
        db_mbar_expect_tx(&bars[slot], SOLVE_FSTAGE_BYTES);
        db_bulk_g2s(st, lu_tile + (int64_t)q * SOLVE_CE * DB_TILE, SOLVE_CE * DB_TILE * 8, &bars[slot]);
        db_bulk_g2s(st + SOLVE_CE * DB_TILE * 8, ctrl_g + (int64_t)q * SOLVE_CTRL_WORDS, SOLVE_CTRL_WORDS * 4, &bars[slot]);
    };
    if (threadIdx.x == 0) {
        for (int i = 0; i < nstages; ++i) db_mbar_init(&bars[i], 1);
        db_mbar_fence_init();
    }
    __syncthreads();
    if (threadIdx.x == 0)
        for (int q = 0; q < nstages && q < nchunks; ++q) issue(q, q);
    if (active) SOLVE_PROLOGUE(NV, B.n)
    auto stage_ctrl = [&](int slot) { return reinterpret_cast<const int*>(ring + (size_t)slot * SOLVE_FSTAGE_BYTES + SOLVE_CE * DB_TILE * 8); };
    int slot = 0;
    unsigned phase = 0;
    double acc = 0.0;
    double xa[SOLVE_CE], xb[SOLVE_CE];
    if (nchunks > 0 && active) { db_mbar_wait(&bars[0], 0); solve_gather(stage_ctrl(0), x, xa); }
    // two chunks per iteration so that the two gather buffers alternate without register copies
    for (int q = 0; q < nchunks; q += 2) {
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int qq = q + half;
            if (qq >= nchunks) break;
            int nslot = slot + 1; unsigned nphase = phase;
            if (nslot == nstages) { nslot = 0; nphase ^= 1; }
            if (active) {
                if (qq + 1 < nchunks) {                              // gather of the NEXT chunk goes out first
                    db_mbar_wait(&bars[nslot], nphase);
                    if (half == 0) solve_gather(stage_ctrl(nslot), x, xb); else solve_gather(stage_ctrl(nslot), x, xa);
                }
                const unsigned char* st = ring + (size_t)slot * SOLVE_FSTAGE_BYTES;
                const double* __restrict__ vals = reinterpret_cast<const double*>(st) + lane;
                const int* __restrict__ ctrl = reinterpret_cast<const int*>(st + SOLVE_CE * DB_TILE * 8);
                if (qq < nfwd) acc = (half == 0) ? solve_chunk_pipe<true>(vals, ctrl, x, xa, acc) : solve_chunk_pipe<true>(vals, ctrl, x, xb, acc);
                else acc = (half == 0) ? solve_chunk_pipe<false>(vals, ctrl, x, xa, acc) : solve_chunk_pipe<false>(vals, ctrl, x, xb, acc);
            }
            __syncthreads();                                   // every warp is done with this stage
            if (threadIdx.x == 0 && qq + nstages < nchunks) issue(qq + nstages, slot);
            slot = nslot; phase = nphase;
        }
    }
}


// ---------------------------------------------------------------------------------------------------------
// Warp-specialised variant of k_batches_solve_flat: a PRODUCER warp feeds the factor ring, the consumer warps never meet
// at a CTA barrier.  In the kernel above every chunk ends with __syncthreads() + thread 0 issuing the next stage
// (mbarrier.arrive.expect_tx + two cp.async.bulk), so all eight warps advance at the pace of warp 0 and pay the issue
// latency of the bulk copies once per chunk: the time per launch then hardly depends on the number of tiles (one thread's
// chain of chunks), i.e. the chain, not the bandwidth, sets the time.
// Here stage release is an arrival-count mbarrier per stage (one arrival per consumer warp), the producer lane waits on
// it before refilling, and consumers only ever wait for "stage full".
// ---------------------------------------------------------------------------------------------------------
template <int NV, int MINB>
__global__ void __launch_bounds__(SOLVE_THREADS * SOLVE_MAX_RHS + 32, MINB)
k_batches_solve_ws(const db_batch* __restrict__ batches, int nbatch, int lu_slot, int x_slot, db_slotcomb rhs, int nstages_pf)
{
    // nstages_pf = ring depth | row-start prefetch mode << 8 | chunks per stage << 16.  A stage carries `cps` consecutive
    // 16-entry chunks (their factor values, then their control blocks): a single thread can only issue a bulk copy every few
    // hundred cycles, so with one chunk per stage the producer lane, not the consumers, paces the sweep.
    const int nstages = nstages_pf & 255, pfmode = (nstages_pf >> 8) & 255, cps = (nstages_pf >> 16) & 255;
    const size_t stage_bytes = (size_t)cps * SOLVE_FSTAGE_BYTES;
    DB_SMEM(unsigned char, ring);
    db_mbar_t* full = reinterpret_cast<db_mbar_t*>(ring + (size_t)nstages * stage_bytes);
    db_mbar_t* empty = full + nstages;
    const int bi = find_batch(batches, nbatch, blockIdx.x, 0);
    const db_batch& B = batches[bi];
    const int tile = blockIdx.x - B.blk_solve;
    const int ncons = blockDim.x - 32;                          // consumer threads: 64 per member group
    const int ngroups = ncons / SOLVE_THREADS;
    const int act_groups = B.nrhs < ngroups ? B.nrhs : ngroups;
    const int nchunks = B.n_entries / SOLVE_CE, nfwd = B.n_fwd / SOLVE_CE;
    const int nst_total = (nchunks + cps - 1) / cps;            // stages to stream
    if (threadIdx.x == 0) {
        for (int i = 0; i < nstages; ++i) {
            db_mbar_init(&full[i], 1);
            db_cbar_init(&empty[i], DB_CBAR_PER_THREAD ? act_groups * SOLVE_THREADS : act_groups * (SOLVE_THREADS / 32));
        }
        db_mbar_fence_init();
    }
    __syncthreads();
    if ((int)threadIdx.x >= ncons) {
        // ---- producer warp: one lane streams the tile's factors + control blocks through the ring
        if (threadIdx.x == ncons) {
            const double* __restrict__ lu_tile = B.lu[lu_slot] + (int64_t)tile * B.n_entries * DB_TILE;
            const int32_t* __restrict__ ctrl_g = B.ctrl;
            int slot = 0;
            unsigned par = 0;                                   // parity of the "empty" phase to wait for: (t / nstages - 1) & 1
            for (int t = 0; t < nst_total; ++t) {
                if (t >= nstages) db_mbar_wait(&empty[slot], par);
                const int q0 = t * cps, cs = (nchunks - q0 < cps) ? nchunks - q0 : cps;
                unsigned char* st = ring + (size_t)slot * stage_bytes;
                db_mbar_expect_tx(&full[slot], (unsigned)(cs * SOLVE_FSTAGE_BYTES));
                db_bulk_g2s(st, lu_tile + (int64_t)q0 * SOLVE_CE * DB_TILE, (unsigned)(cs * SOLVE_CE * DB_TILE * 8), &full[slot]);
                db_bulk_g2s(st + (size_t)cps * SOLVE_CE * DB_TILE * 8, ctrl_g + (int64_t)q0 * SOLVE_CTRL_WORDS, (unsigned)(cs * SOLVE_CTRL_WORDS * 4), &full[slot]);
                if (++slot == nstages) { slot = 0; if (t >= nstages) par ^= 1; }      // flips at the end of every wrap after the first
            }
        }
        return;
    }
    const int grp = threadIdx.x / SOLVE_THREADS, lane = threadIdx.x % SOLVE_THREADS;
    if (grp >= B.nrhs) return;                                  // member groups this batch does not have
    const int s = grp * B.ld + tile * SOLVE_THREADS + lane;      // padded lanes run on the zero padding
    const int64_t tb = db_tbase(s, B.n);
    double* x = B.vec[x_slot] + tb;
    const double* rv[NV];
    double cf[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) { rv[j] = B.vec[rhs.slot[j < rhs.nvec ? j : 0]] + tb; cf[j] = (j < rhs.nvec) ? rhs.coef[j] : 0.0; }
    SOLVE_PROLOGUE(NV, B.n)
    double acc = 0.0;
    int slot = 0;
    unsigned phase = 0;
    for (int t = 0; t < nst_total; ++t) {
        db_mbar_wait(&full[slot], phase);
        const unsigned char* st = ring + (size_t)slot * stage_bytes;
        const int q0 = t * cps, cs = (nchunks - q0 < cps) ? nchunks - q0 : cps;
        for (int c = 0; c < cs; ++c) {
            const int q = q0 + c;
            const double* __restrict__ vals = reinterpret_cast<const double*>(st + (size_t)c * SOLVE_CE * DB_TILE * 8) + lane;
            const int* __restrict__ ctrl = reinterpret_cast<const int*>(st + (size_t)cps * SOLVE_CE * DB_TILE * 8) + c * SOLVE_CTRL_WORDS;
            const unsigned mB = (unsigned)ctrl[2 * SOLVE_CE + 1], mF = (unsigned)ctrl[2 * SOLVE_CE + 2];
            solve_prefetch(ctrl, x, pfmode & 3);
            if ((mB | mF) == 0) acc = solve_chunk_pure(vals, ctrl, x, acc);
            else if (q < nfwd) acc = mF ? solve_chunk_flat<true, true>(vals, ctrl, x, acc) : solve_chunk_flat<true, false>(vals, ctrl, x, acc);
            else acc = mF ? solve_chunk_flat<false, true>(vals, ctrl, x, acc) : solve_chunk_flat<false, false>(vals, ctrl, x, acc);
        }
#if DB_CBAR_PER_THREAD
        db_cbar_arrive(&empty[slot]);
#else
        __syncwarp();
        if ((threadIdx.x & 31) == 0) db_cbar_arrive(&empty[slot]);
#endif
        if (++slot == nstages) { slot = 0; phase ^= 1; }
    }
}

// ---------------------------------------------------------------------------------------------------------
// Members in registers (DB_SOLVE_RT = 2 / 4): one thread carries RT members of its pencil -- RT independent recurrences
// driven by the same factor values and the same control block.  The sweep is latency-bound (one dependent chain per
// thread: mbarrier -> control words -> 16 gathers from L2 -> 16 dependent FMAs; with few tiles per GPU -- strong scaling
// over several GPUs -- the time per launch stops shrinking at the length of that chain).  RT chains per thread put RT x the loads in flight per warp and amortise
// the shared-memory reads of the factor values and of the control block over RT systems.  Gathers are issued per half
// chunk (8 entries x RT members) to bound the register count.  Work vectors are allocated for SOLVE_MAX_RHS members per
// batch (missing members are all-zero columns: they are solved along, never read), so there is no per-member predicate.
// ---------------------------------------------------------------------------------------------------------
template <bool FWD, bool LATE, int RT>
__device__ __forceinline__ void solve_chunk_mr(const double* __restrict__ vals, const int* __restrict__ ctrl, double* const (&x)[RT], double (&acc)[RT])
{
    const unsigned maskE = (unsigned)ctrl[2 * SOLVE_CE], maskB = (unsigned)ctrl[2 * SOLVE_CE + 1], maskF = (unsigned)ctrl[2 * SOLVE_CE + 2];
#pragma unroll
    for (int h = 0; h < SOLVE_CE; h += 8) {
        int goff[8], foff[8];
#pragma unroll
        for (int j = 0; j < 8; j += 4) {
            const int4 g = *reinterpret_cast<const int4*>(ctrl + h + j);
            goff[j] = g.x; goff[j + 1] = g.y; goff[j + 2] = g.z; goff[j + 3] = g.w;
        }
        double xv[8][RT];
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int r = 0; r < RT; ++r) xv[j][r] = x[r][goff[j]];
#pragma unroll
        for (int j = 0; j < 8; j += 4) {
            const int4 f = *reinterpret_cast<const int4*>(ctrl + SOLVE_CE + h + j);
            foff[j] = f.x; foff[j + 1] = f.y; foff[j + 2] = f.z; foff[j + 3] = f.w;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const double v = vals[(h + j) * DB_TILE];
            const unsigned bit = 1u << (h + j);
#pragma unroll
            for (int r = 0; r < RT; ++r) {
                if (LATE) { if (maskF & bit) xv[j][r] = x[r][goff[j]]; }
                const double acc_a = fma(-v, xv[j][r], acc[r]);
                const double val = FWD ? acc[r] : acc[r] * v;
                if (maskE & bit) x[r][foff[j]] = val;
                acc[r] = (maskB & bit) ? xv[j][r] : acc_a;
            }
        }
    }
}

template <int RT>
__device__ __forceinline__ void solve_chunk_mr_pure(const double* __restrict__ vals, const int* __restrict__ ctrl, double* const (&x)[RT], double (&acc)[RT])
{
#pragma unroll
    for (int h = 0; h < SOLVE_CE; h += 8) {
        double xv[8][RT];
#pragma unroll
        for (int j = 0; j < 8; j += 4) {
            const int4 g = *reinterpret_cast<const int4*>(ctrl + h + j);
#pragma unroll
            for (int r = 0; r < RT; ++r) { xv[j][r] = x[r][g.x]; xv[j + 1][r] = x[r][g.y]; xv[j + 2][r] = x[r][g.z]; xv[j + 3][r] = x[r][g.w]; }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const double v = vals[(h + j) * DB_TILE];
#pragma unroll
            for (int r = 0; r < RT; ++r) acc[r] = fma(-v, xv[j][r], acc[r]);
        }
    }
}

template <int NV, int RT>
__global__ void __launch_bounds__(SOLVE_THREADS * SOLVE_MAX_RHS / RT)
k_batches_solve_mr(const db_batch* __restrict__ batches, int nbatch, int lu_slot, int x_slot, db_slotcomb rhs, int nstages)
{
    DB_SMEM(unsigned char, ring);
    db_mbar_t* bars = reinterpret_cast<db_mbar_t*>(ring + (size_t)nstages * SOLVE_FSTAGE_BYTES);
    const int bi = find_batch(batches, nbatch, blockIdx.x, 0);
    const db_batch& B = batches[bi];
    const int tile = blockIdx.x - B.blk_solve;
    const int grp = threadIdx.x / SOLVE_THREADS, lane = threadIdx.x % SOLVE_THREADS;
    const bool active = grp * RT < B.nrhs;                      // groups beyond the batch's members only take part in the barriers
    const double* __restrict__ lu_tile = B.lu[lu_slot] + (int64_t)tile * B.n_entries * DB_TILE;
    const int32_t* __restrict__ ctrl_g = B.ctrl;
    const int nchunks = B.n_entries / SOLVE_CE, nfwd = B.n_fwd / SOLVE_CE;
    int64_t tb[RT];
    double* x[RT];
#pragma unroll
    for (int r = 0; r < RT; ++r) {
        tb[r] = db_tbase(((active ? grp : 0) * RT + r) * B.ld + tile * SOLVE_THREADS + lane, B.n);
        x[r] = B.vec[x_slot] + tb[r];
    }
    auto issue = [&](int q, int slot) {
        unsigned char* st = ring + (size_t)slot * SOLVE_FSTAGE_BYTES;
        db_mbar_expect_tx(&bars[slot], SOLVE_FSTAGE_BYTES);
        db_bulk_g2s(st, lu_tile + (int64_t)q * SOLVE_CE * DB_TILE, SOLVE_CE * DB_TILE * 8, &bars[slot]);
        db_bulk_g2s(st + SOLVE_CE * DB_TILE * 8, ctrl_g + (int64_t)q * SOLVE_CTRL_WORDS, SOLVE_CTRL_WORDS * 4, &bars[slot]);
    };
    if (threadIdx.x == 0) {
        for (int i = 0; i < nstages; ++i) db_mbar_init(&bars[i], 1);
        db_mbar_fence_init();
    }
    __syncthreads();
    if (threadIdx.x == 0)
        for (int q = 0; q < nstages && q < nchunks; ++q) issue(q, q);
    if (active) {
        // right-hand side: x <- sum_q coef[q] vec[q], RT * NV independent loads in flight per row
        const int nv = rhs.nvec < NV ? rhs.nvec : NV;
        for (int i = 0; i < B.n; ++i) {
            double a_[RT];
#pragma unroll
            for (int r = 0; r < RT; ++r) a_[r] = 0.0;
#pragma unroll
            for (int q = 0; q < NV; ++q) {
                if (q < nv) {
                    const double* __restrict__ v = B.vec[rhs.slot[q]];
                    const double c = rhs.coef[q];
#pragma unroll
                    for (int r = 0; r < RT; ++r) a_[r] = fma(c, DB_LDCS(v + tb[r] + (int64_t)i * DB_TILE), a_[r]);
                }
            }
#pragma unroll
            for (int r = 0; r < RT; ++r) x[r][(int64_t)i * DB_TILE] = a_[r];
        }
    }
    int slot = 0;
    unsigned phase = 0;
    double acc[RT];
#pragma unroll
    for (int r = 0; r < RT; ++r) acc[r] = 0.0;
    for (int q = 0; q < nchunks; ++q) {
        if (active) {
            db_mbar_wait(&bars[slot], phase);
            const unsigned char* st = ring + (size_t)slot * SOLVE_FSTAGE_BYTES;
            const double* __restrict__ vals = reinterpret_cast<const double*>(st) + lane;
            const int* __restrict__ ctrl = reinterpret_cast<const int*>(st + SOLVE_CE * DB_TILE * 8);
            const unsigned mB = (unsigned)ctrl[2 * SOLVE_CE + 1], mF = (unsigned)ctrl[2 * SOLVE_CE + 2];
            if ((mB | mF) == 0) solve_chunk_mr_pure<RT>(vals, ctrl, x, acc);
            else if (q < nfwd) { if (mF) solve_chunk_mr<true, true, RT>(vals, ctrl, x, acc); else solve_chunk_mr<true, false, RT>(vals, ctrl, x, acc); }
            else { if (mF) solve_chunk_mr<false, true, RT>(vals, ctrl, x, acc); else solve_chunk_mr<false, false, RT>(vals, ctrl, x, acc); }
        }
        if (blockDim.x > 32) __syncthreads(); else __syncwarp();        // every warp is done with this stage
        if (threadIdx.x == 0 && q + nstages < nchunks) issue(q + nstages, slot);
        if (++slot == nstages) { slot = 0; phase ^= 1; }
    }
}


// ---------------------------------------------------------------------------------------------------------
// Deep-prefetch variant for the latency-bound regime (few tiles per GPU: 8-GPU strong scaling, where the time of the
// kernels above stops shrinking at the length of ONE thread's dependent chain: per 16-entry chunk an L2 round trip for the
// gathers, ~1 us, then 16 dependent FMAs).  Here the 16 gathers of chunk q + D are issued while chunk q is consumed -- as
// 8-byte cp.async (LDGSTS) copies into a per-thread column of a shared-memory ring, so they cost no registers and D chunks
// of gathers are in flight per thread.  Values whose source row is finished AFTER the gather was issued (15 % of the
// entries at D = 3 with the level-ordered stream) come from a second shared-memory ring holding the last SOLVE_DEEP_RRN
// finished rows of every thread (control words 36..40, pencils.py solve_control_blocks); the rare older ones are re-read
// from global memory.  One 256-thread CTA per SM (194 KB of shared memory).
// ---------------------------------------------------------------------------------------------------------
#define SOLVE_DEEP_D 3
#define SOLVE_DEEP_RRN 16
template <int NV>
__global__ void __launch_bounds__(SOLVE_THREADS * SOLVE_MAX_RHS, 1)
k_batches_solve_deep(const db_batch* __restrict__ batches, int nbatch, int lu_slot, int x_slot, db_slotcomb rhs, int nstages_pf)
{
    const int nstages = nstages_pf & 255, pfmode = nstages_pf >> 8;
    constexpr int D = SOLVE_DEEP_D, GS = D + 1, RRN = SOLVE_DEEP_RRN;
    DB_SMEM(unsigned char, ring);
    const int NT = blockDim.x;
    db_mbar_t* bars = reinterpret_cast<db_mbar_t*>(ring + (size_t)nstages * SOLVE_FSTAGE_BYTES);
    double* G = reinterpret_cast<double*>(ring + (((size_t)nstages * SOLVE_FSTAGE_BYTES + (size_t)nstages * sizeof(db_mbar_t) + 15) & ~(size_t)15));
    double* RR = G + (size_t)GS * SOLVE_CE * NT;                 // [RRN][NT]
    const int bi = find_batch(batches, nbatch, blockIdx.x, 0);
    const db_batch& B = batches[bi];
    const int tile = blockIdx.x - B.blk_solve;
    // blockDim.x = 64 * (members per CTA); blockIdx.y selects the member group (the members of a tile may be spread over
    // several CTAs, each with its own factor ring, so that more SMs work when there are few tiles)
    const int grp = blockIdx.y * (blockDim.x / SOLVE_THREADS) + threadIdx.x / SOLVE_THREADS, lane = threadIdx.x % SOLVE_THREADS;
    if (blockIdx.y * (blockDim.x / SOLVE_THREADS) >= B.nrhs) return;      // whole CTA without members
    const bool active = grp < B.nrhs;
    const int s = (active ? grp : 0) * B.ld + tile * SOLVE_THREADS + lane;
    const int64_t tb = db_tbase(s, B.n);
    const double* __restrict__ lu_tile = B.lu[lu_slot] + (int64_t)tile * B.n_entries * DB_TILE;
    const int32_t* __restrict__ ctrl_g = B.ctrl;
    const int nchunks = B.n_entries / SOLVE_CE, nfwd = B.n_fwd / SOLVE_CE;
    double* x = B.vec[x_slot] + tb;
    const double* rv[NV];
    double cf[NV];
#pragma unroll
    for (int j = 0; j < NV; ++j) { rv[j] = B.vec[rhs.slot[j < rhs.nvec ? j : 0]] + tb; cf[j] = (j < rhs.nvec) ? rhs.coef[j] : 0.0; }
    auto issue = [&](int q, int slot) {
        unsigned char* st = ring + (size_t)slot * SOLVE_FSTAGE_BYTES;
        db_mbar_expect_tx(&bars[slot], SOLVE_FSTAGE_BYTES);
        db_bulk_g2s(st, lu_tile + (int64_t)q * SOLVE_CE * DB_TILE, SOLVE_CE * DB_TILE * 8, &bars[slot]);
        db_bulk_g2s(st + SOLVE_CE * DB_TILE * 8, ctrl_g + (int64_t)q * SOLVE_CTRL_WORDS, SOLVE_CTRL_WORDS * 4, &bars[slot]);
    };
    if (threadIdx.x == 0) {
        for (int i = 0; i < nstages; ++i) db_mbar_init(&bars[i], 1);
        db_mbar_fence_init();
    }
    __syncthreads();
    if (threadIdx.x == 0)
        for (int q = 0; q < nstages && q < nchunks; ++q) issue(q, q);
    if (active) SOLVE_PROLOGUE(NV, B.n)
    auto stage_ctrl = [&](int slot) { return reinterpret_cast<const int*>(ring + (size_t)slot * SOLVE_FSTAGE_BYTES + SOLVE_CE * DB_TILE * 8); };
    // gathers of chunk q -> G[q % GS][j][thread]; the stage of chunk q is slot q % nstages, its first phase parity (q / nstages) & 1
    auto gather = [&](int q) {
        const int slot = q % nstages;
        db_mbar_wait(&bars[slot], (unsigned)((q / nstages) & 1));
        const int* __restrict__ ctrl = stage_ctrl(slot);
        double* g = G + ((size_t)(q % GS) * SOLVE_CE) * NT + threadIdx.x;
#pragma unroll
        for (int j = 0; j < SOLVE_CE; j += 4) {
            const int4 o = *reinterpret_cast<const int4*>(ctrl + j);
            db_cp_async8(g + (size_t)(j + 0) * NT, x + o.x); db_cp_async8(g + (size_t)(j + 1) * NT, x + o.y);
            db_cp_async8(g + (size_t)(j + 2) * NT, x + o.z); db_cp_async8(g + (size_t)(j + 3) * NT, x + o.w);
        }
    };
    if (active)
        for (int q = 0; q < D; ++q) { if (q < nchunks) gather(q); db_cp_commit(); }
    unsigned cnt = 0;                                           // row ends so far (uniform): next slot of the recent-rows ring
    double acc = 0.0;
    double* rr = RR + threadIdx.x;
    for (int q = 0; q < nchunks; ++q) {
        const int slot = q % nstages;
        if (active) {
            if (q + D < nchunks) gather(q + D);
            db_cp_commit();
            db_cp_wait<D>();                                     // the group of chunk q (and everything older) has landed
            const unsigned char* st = ring + (size_t)slot * SOLVE_FSTAGE_BYTES;
            const double* __restrict__ vals = reinterpret_cast<const double*>(st) + lane;
            const int* __restrict__ ctrl = reinterpret_cast<const int*>(st + SOLVE_CE * DB_TILE * 8);
            const double* g = G + ((size_t)(q % GS) * SOLVE_CE) * NT + threadIdx.x;
            const unsigned maskE = (unsigned)ctrl[32], maskB = (unsigned)ctrl[33], maskR = (unsigned)ctrl[36], maskG = (unsigned)ctrl[37];
            const bool fwd = q < nfwd;
            solve_prefetch(ctrl, x, pfmode);
            if ((maskE | maskB | maskR | maskG) == 0) {
#pragma unroll
                for (int j = 0; j < SOLVE_CE; ++j) acc = fma(-vals[j * DB_TILE], g[(size_t)j * NT], acc);
            } else {
                const unsigned rs0 = (unsigned)ctrl[38], rs1 = (unsigned)ctrl[39], rs2 = (unsigned)ctrl[40];
#pragma unroll
                for (int j = 0; j < SOLVE_CE; ++j) {
                    const unsigned bit = 1u << j;
                    const double v = vals[j * DB_TILE];
                    double xv = g[(size_t)j * NT];
                    if (maskR & bit) {
                        const unsigned w = (j < 6) ? rs0 : (j < 12) ? rs1 : rs2;
                        xv = rr[(size_t)((w >> (5 * (j % 6))) & 31u) * NT];
                    }
                    if (maskG & bit) xv = x[ctrl[j]];
                    const double acc_a = fma(-v, xv, acc);
                    const double val = fwd ? acc : acc * v;
                    if (maskE & bit) { x[ctrl[SOLVE_CE + j]] = val; rr[(size_t)(cnt & (RRN - 1)) * NT] = val; ++cnt; }
                    acc = (maskB & bit) ? xv : acc_a;
                }
            }
        }
        if (blockDim.x > 32) __syncthreads(); else __syncwarp();     // every warp is done with this stage
        if (threadIdx.x == 0 && q + nstages < nchunks) issue(q + nstages, slot);
    }
}

// Run-time choice of the solve kernel and its ring (db_batches_solve_set_mode); a negative field keeps the environment's choice.
// Kernels: 0 k_batches_solve_ws, 1 _flat, 2 _pipe, 3 _mr<2>, 4 _mr<4>, 5 _deep.
static int g_sv_kernel = -1, g_sv_stages = -1, g_sv_cps = -1, g_sv_minb = -1, g_sv_pf = -1, g_sv_mpc = -1;
#define SOLVE_WS_SMEM(nst, cps) ((size_t)(nst) * (cps) * SOLVE_FSTAGE_BYTES + (size_t)2 * (nst) * sizeof(db_mbar_t))

extern "C" int db_batches_solve_set_mode(int32_t kernel, int32_t stages, int32_t chunks_per_stage, int32_t minb, int32_t prefetch,
                                         int32_t deep_members)
{
    if (kernel > 5 || (stages >= 0 && (stages < 2 || stages > 24)) || chunks_per_stage == 0 || chunks_per_stage > 8 || minb == 0 ||
        minb > 4 || prefetch > 2 || (deep_members >= 0 && deep_members != 1 && deep_members != 2 && deep_members != 4)) {
        db_set_error("batches_solve_set_mode: argument out of range (kernel %d, stages %d, chunks per stage %d, minb %d, prefetch %d, "
                     "deep members %d)", kernel, stages, chunks_per_stage, minb, prefetch, deep_members);
        return 1;
    }
    if (kernel == 5 && stages >= 0 && stages < SOLVE_DEEP_D + 2) {
        db_set_error("batches_solve_set_mode: the deep kernel needs at least %d stages", SOLVE_DEEP_D + 2); return 1;
    }
    if (kernel == 0 && stages >= 0 && chunks_per_stage > 0 && SOLVE_WS_SMEM(stages, chunks_per_stage) > DB_MAX_SMEM) {
        db_set_error("batches_solve_set_mode: %d stages of %d chunks need %zu bytes of shared memory (limit %d)", stages,
                     chunks_per_stage, SOLVE_WS_SMEM(stages, chunks_per_stage), DB_MAX_SMEM);
        return 1;
    }
    g_sv_kernel = kernel; g_sv_stages = stages; g_sv_cps = chunks_per_stage; g_sv_minb = minb; g_sv_pf = prefetch; g_sv_mpc = deep_members;
    return 0;
}

extern "C" int db_batches_solve(const db_batch* batches, int32_t nbatch, int32_t total_blocks, int32_t max_nrhs, int32_t lu_slot, int32_t x_slot,
                                const db_slotcomb* rhs, void* stream)
{
    if (nbatch <= 0 || total_blocks <= 0) return 0;
    // nvec >= 1: the kernels pad the combination to their template size with zero-coefficient copies of the first term, so an
    // empty one would give 0 * vec[slot[0]] (NaN where that slot holds NaN) in some variants and 0 in others
    if (rhs->nvec < 1 || rhs->nvec > 16 || lu_slot < 0 || lu_slot >= DB_MAX_LU || max_nrhs < 1 || max_nrhs > SOLVE_MAX_RHS) {
        db_set_error("batches_solve: bad arguments"); return 1;
    }
    const dim3 g(total_blocks), b(SOLVE_THREADS * max_nrhs);
    const int nv = rhs->nvec;
    static int st_env = -1, pipe_env = 0, rt_env = 0, minb_env = 3, deep_env = -1, ws_env = 1, pf_env = 2, cps_env = 2;
    if (st_env < 0) {
        const char* t = getenv("DB_SOLVE_STAGES"); st_env = t ? atoi(t) : 0;
        const char* p = getenv("DB_SOLVE_PIPE"); pipe_env = p ? atoi(p) : 0;
        const char* r = getenv("DB_SOLVE_RT"); rt_env = r ? atoi(r) : 0;
        const char* m = getenv("DB_SOLVE_MINB"); minb_env = m ? atoi(m) : 3;
        const char* d = getenv("DB_SOLVE_DEEP"); deep_env = d ? atoi(d) : -1;
        const char* w = getenv("DB_SOLVE_WS"); ws_env = w ? atoi(w) : 1;
        const char* f = getenv("DB_SOLVE_PF"); pf_env = f ? atoi(f) : 2;
        const char* c = getenv("DB_SOLVE_CPS"); cps_env = c ? atoi(c) : 2;
        if (cps_env < 1 || cps_env > 8) cps_env = 2;
    }
    // fields set by db_batches_solve_set_mode replace the environment's
    const int st_sel = g_sv_stages >= 0 ? g_sv_stages : st_env;
    const int cps = g_sv_cps > 0 ? g_sv_cps : cps_env, minb = g_sv_minb > 0 ? g_sv_minb : minb_env, pf = g_sv_pf >= 0 ? g_sv_pf : pf_env;
    // ring depth: with ~7 CTAs per SM two stages already keep 100+ KB of factor bytes in flight per SM and every
    // further stage only shrinks the L1 the x gathers live in; with few CTAs per SM the ring is the only source of
    // memory parallelism, so it gets deep
    const int per_sm = (total_blocks + db_num_sms() - 1) / db_num_sms();
    int nst = per_sm >= 5 ? 2 : per_sm >= 3 ? 4 : per_sm >= 2 ? 8 : 16;
    if (st_sel >= 2 && st_sel <= 24) nst = st_sel;
    const size_t smem = (size_t)nst * SOLVE_FSTAGE_BYTES + (size_t)nst * sizeof(db_mbar_t);
    // members per thread: 1 = k_batches_solve_flat; 2 / 4 = k_batches_solve_mr (RT chains per thread; opt-in, DB_SOLVE_RT)
    int rt = rt_env ? rt_env : 1;       // 2 and 4 leave fewer resident warps
    if (rt != 1 && rt != 2 && rt != 4) rt = 1;
    if (rt > max_nrhs) rt = max_nrhs >= 2 ? 2 : 1;
    // deep-prefetch kernel: by default when there is at most one tile per SM (the launch is then bound by one thread's
    // dependent chain, not by bandwidth); DB_SOLVE_DEEP = 0 / 1 forces it off / on.  Members per CTA: as few as still give
    // at most one CTA per SM (more SMs at work, deeper factor ring per CTA); DB_SOLVE_DEEP_MPC overrides.
    const bool deep = deep_env > 0;          // opt-in (DB_SOLVE_DEEP=1)
    int kern = g_sv_kernel;
    if (kern < 0) kern = (ws_env && !deep && rt == 1 && !pipe_env) ? 0 : deep ? 5 : (rt == 4 && !pipe_env) ? 4 : (rt == 2 && !pipe_env) ? 3
                       : pipe_env ? 2 : 1;
    else if (kern == 3 || kern == 4) rt = kern == 3 ? 2 : 4;      // as asked: the work vectors hold whole groups of 4 members
    const dim3 bmr(SOLVE_THREADS * ((max_nrhs + rt - 1) / rt));
    static int mpc_env = -1;
    if (mpc_env < 0) { const char* e = getenv("DB_SOLVE_DEEP_MPC"); mpc_env = e ? atoi(e) : 0; }
    const int mpc_sel = g_sv_mpc > 0 ? g_sv_mpc : mpc_env;
    int mpc = 1;
    while (mpc < max_nrhs && total_blocks * ((max_nrhs + mpc - 1) / mpc) > db_num_sms()) mpc *= 2;
    if (mpc_sel == 1 || mpc_sel == 2 || mpc_sel == 4) mpc = mpc_sel;
    if (mpc > max_nrhs) mpc = max_nrhs;
    const dim3 g_deep(total_blocks, (max_nrhs + mpc - 1) / mpc), b_deep(SOLVE_THREADS * mpc);
    const size_t deep_fixed = (size_t)((SOLVE_DEEP_D + 1) * SOLVE_CE + SOLVE_DEEP_RRN) * b_deep.x * sizeof(double) + 64;
    int nst_deep = (int)(((size_t)220 * 1024 - deep_fixed) / (SOLVE_FSTAGE_BYTES + sizeof(db_mbar_t)));
    if (nst_deep > 24) nst_deep = 24;
    if (kern == 5 && g_sv_stages >= 0 && g_sv_stages > nst_deep) {
        db_set_error("batches_solve: %d stages of the deep kernel do not fit in shared memory next to %d members per CTA (at most %d)",
                     g_sv_stages, mpc, nst_deep);
        return 1;
    }
    if (st_sel >= SOLVE_DEEP_D + 2 && st_sel <= 24 && (st_sel < nst_deep || st_sel == g_sv_stages)) nst_deep = st_sel;
    const size_t smem_deep = (((size_t)nst_deep * SOLVE_FSTAGE_BYTES + (size_t)nst_deep * sizeof(db_mbar_t) + 15) & ~(size_t)15) + deep_fixed;
    int nst_ws = (nst * 1 + cps - 1) / cps; if (nst_ws < 3) nst_ws = 3;
    if (st_sel >= 2 && st_sel <= 24) nst_ws = st_sel;
    const size_t smem_ws = SOLVE_WS_SMEM(nst_ws, cps);
    if (kern == 0 && smem_ws > DB_MAX_SMEM) {
        db_set_error("batches_solve: %d stages of %d chunks need %zu bytes of shared memory (limit %d)", nst_ws, cps, smem_ws, DB_MAX_SMEM);
        return 1;
    }
#define FLAT_GO(NV_) { static int attr_st = 0; \
    if (!attr_st) { DB_SET_SMEM_ATTR((k_batches_solve_flat<NV_, 2>)); DB_SET_SMEM_ATTR((k_batches_solve_flat<NV_, 3>)); DB_SET_SMEM_ATTR((k_batches_solve_flat<NV_, 4>)); \
                    DB_SET_SMEM_ATTR((k_batches_solve_pipe<NV_>)); \
                    DB_SET_SMEM_ATTR((k_batches_solve_mr<NV_, 2>)); DB_SET_SMEM_ATTR((k_batches_solve_mr<NV_, 4>)); \
                    DB_SET_SMEM_ATTR((k_batches_solve_ws<NV_, 1>)); DB_SET_SMEM_ATTR((k_batches_solve_ws<NV_, 2>)); DB_SET_SMEM_ATTR((k_batches_solve_ws<NV_, 3>)); \
                    DB_SET_SMEM_ATTR((k_batches_solve_deep<NV_>)); attr_st = 1; } \
    if (kern == 0) { \
        const int code = nst_ws | (pf << 8) | (cps << 16); \
        if (minb == 4) DB_LAUNCH((k_batches_solve_ws<NV_, 3>), g, dim3(b.x + 32), smem_ws, stream, batches, nbatch, lu_slot, x_slot, *rhs, code); \
        else if (minb == 1) DB_LAUNCH((k_batches_solve_ws<NV_, 1>), g, dim3(b.x + 32), smem_ws, stream, batches, nbatch, lu_slot, x_slot, *rhs, code); \
        else DB_LAUNCH((k_batches_solve_ws<NV_, 2>), g, dim3(b.x + 32), smem_ws, stream, batches, nbatch, lu_slot, x_slot, *rhs, code); } \
    else if (kern == 5) DB_LAUNCH((k_batches_solve_deep<NV_>), g_deep, b_deep, smem_deep, stream, batches, nbatch, lu_slot, x_slot, *rhs, nst_deep | (pf << 8)); \
    else if (kern == 4) DB_LAUNCH((k_batches_solve_mr<NV_, 4>), g, bmr, smem, stream, batches, nbatch, lu_slot, x_slot, *rhs, nst); \
    else if (kern == 3) DB_LAUNCH((k_batches_solve_mr<NV_, 2>), g, bmr, smem, stream, batches, nbatch, lu_slot, x_slot, *rhs, nst); \
    else if (kern == 2) DB_LAUNCH((k_batches_solve_pipe<NV_>), g, b, smem, stream, batches, nbatch, lu_slot, x_slot, *rhs, nst); \
    else if (minb == 4) DB_LAUNCH((k_batches_solve_flat<NV_, 4>), g, b, smem, stream, batches, nbatch, lu_slot, x_slot, *rhs, nst | (pf << 8)); \
    else if (minb == 2) DB_LAUNCH((k_batches_solve_flat<NV_, 2>), g, b, smem, stream, batches, nbatch, lu_slot, x_slot, *rhs, nst | (pf << 8)); \
    else DB_LAUNCH((k_batches_solve_flat<NV_, 3>), g, b, smem, stream, batches, nbatch, lu_slot, x_slot, *rhs, nst | (pf << 8)); }
    if (nv <= 1) FLAT_GO(1) else if (nv == 2) FLAT_GO(2) else if (nv == 3) FLAT_GO(3) else if (nv == 4) FLAT_GO(4)
    else if (nv == 5) FLAT_GO(5) else if (nv == 6) FLAT_GO(6) else if (nv <= 8) FLAT_GO(8) else if (nv <= 12) FLAT_GO(12) else FLAT_GO(16)
#undef FLAT_GO
    return db_check_launch("batches_solve");
}

#define MV_MAX_MONO 16
struct MvTerm { double val; int col_off; int mono; };
__device__ __forceinline__ MvTerm mv_load_shared(const db_term* rec, int t)
{
    // staged records: one 16-byte shared-memory load (broadcast: every lane reads the same record)
#ifdef DB_EMU
    MvTerm r; r.val = rec[t].val; r.col_off = rec[t].col_off; r.mono = rec[t].mono; return r;
#else
    const int4 raw = *reinterpret_cast<const int4*>(rec + t);
    MvTerm r; r.val = __hiloint2double(raw.y, raw.x); r.col_off = raw.z; r.mono = raw.w; return r;
#endif
}
__device__ __forceinline__ MvTerm mv_load(const db_term* __restrict__ rec, int t)
{
    // one 16-byte load (the records are 16-byte aligned: the array comes from its own allocation)
#ifdef DB_EMU
    MvTerm r; r.val = rec[t].val; r.col_off = rec[t].col_off; r.mono = rec[t].mono; return r;
#else
    const int4 raw = __ldg(reinterpret_cast<const int4*>(rec) + t);
    MvTerm r; r.val = __hiloint2double(raw.y, raw.x); r.col_off = raw.z; r.mono = raw.w; return r;
#endif
}
// y = (sum_m mono_m T_m) x for the M and L templates of all batches.  One CTA = one 64-system tile x MV_R consecutive rows,
// 256 threads = 4 row groups x 64 systems.  The operators are banded in the mode-major row / column order, so the x rows
// a row block needs form a window of ~2 MV_R rows: it is staged ONCE in shared memory (16-byte cp.async) together with the
// block's term records and the tile's monomial values, and the term loop then runs entirely out of shared memory instead
// of re-reading x through L2 behind long-scoreboard stalls.  The few terms
// outside the window (dense boundary rows) read x from global memory.
#define MV_R 32
#define MV_GROUPS 8
#define MV_THREADS (32 * MV_GROUPS)
#define MV_WMAX 80
#define MV_RECMAX 768
#define MV_SMEM_BYTES ((MV_WMAX * 64 + MV_MAX_MONO * 64) * 8 + MV_RECMAX * 16)
__global__ void __launch_bounds__(MV_THREADS)
k_batches_matvec(const db_batch* __restrict__ batches, int nbatch, int x_slot, int ym_slot, int yl_slot)
{
    // thread = (row group g, system pair sp): the two systems 2 sp, 2 sp + 1 of the tile are adjacent in every array,
    // so each term costs one 16-byte record load, one 16-byte x load and one 16-byte monomial load for two systems
    DB_SMEM(double, win);                                   // [MV_WMAX][64] x window, then monomials [MV_MAX_MONO][64], then records
    double* monos = win + MV_WMAX * 64;
    db_term* recs = reinterpret_cast<db_term*>(monos + MV_MAX_MONO * 64);
    const int bi = find_batch(batches, nbatch, blockIdx.x, 1);
    const db_batch& B = batches[bi];
    const int local = blockIdx.x - B.blk_matvec;
    const int ptiles = (B.S + 63) / 64;                       // tiles of pencils; tiles of vector columns = nrhs * ptiles
    const int tiles = ptiles * B.nrhs;
    const int tile = local % tiles, rb = local / tiles;
    const int ptile = tile % ptiles;                          // pencil tile (monomials are per pencil)
    const int n = B.n, ld = B.ld;
    const int r0 = rb * MV_R, r1 = (r0 + MV_R < n) ? r0 + MV_R : n;
    const int tid = threadIdx.x, sp = tid & 31, g = tid >> 5;
    const int64_t tile_base = (int64_t)tile * n * DB_TILE;
    const double* __restrict__ xt = B.vec[x_slot] + tile_base;
    const int w0 = B.mv_win[2 * rb], wl = B.mv_win[2 * rb + 1];
    const bool do_m = ym_slot >= 0, do_l = yl_slot >= 0;
    const int m0 = B.m_ptr[r0], m1 = B.m_ptr[r1], l0 = B.l_ptr[r0], l1 = B.l_ptr[r1];
    const int nm_rec = do_m ? m1 - m0 : 0, nl_rec = do_l ? l1 - l0 : 0;
    const bool staged = nm_rec + nl_rec <= MV_RECMAX;
    // ---- stage: x window (16-byte chunks), monomials of this tile, term records
    for (int idx = tid; idx < wl * 32; idx += MV_THREADS)
        db_cp_async16(win + 2 * idx, xt + (int64_t)w0 * DB_TILE + 2 * idx);
    const int nm = B.n_mono < MV_MAX_MONO ? B.n_mono : MV_MAX_MONO;
    for (int idx = tid; idx < nm * 32; idx += MV_THREADS)
        db_cp_async16(monos + 2 * idx, B.mono + (int64_t)(idx >> 5) * ld + ptile * 64 + 2 * (idx & 31));
    if (staged) {
        for (int idx = tid; idx < nm_rec; idx += MV_THREADS) db_cp_async16(recs + idx, B.m_rec + m0 + idx);
        for (int idx = tid; idx < nl_rec; idx += MV_THREADS) db_cp_async16(recs + nm_rec + idx, B.l_rec + l0 + idx);
    }
    db_cp_commit();
    db_cp_wait<0>();
    __syncthreads();
    const double2* xs = reinterpret_cast<const double2*>(win) + sp;           // row stride 32 double2
    const double2* ms = reinterpret_cast<const double2*>(monos) + sp;
    const double* __restrict__ xg = xt + 2 * sp;
    for (int which = 0; which < 2; ++which) {
        const int slot = which ? yl_slot : ym_slot;
        if (slot < 0) continue;
        const int32_t* __restrict__ ptr = which ? B.l_ptr : B.m_ptr;
        const int32_t* __restrict__ split = which ? B.l_split : B.m_split;
        const db_term* __restrict__ grec = which ? B.l_rec : B.m_rec;
        const db_term* srec = recs + (which ? nm_rec - l0 : -m0);               // staged copy, indexed like the global array
        double* __restrict__ y = B.vec[slot] + tile_base + 2 * sp;
        for (int i = r0 + g; i < r1; i += MV_GROUPS) {
            const int ta = ptr[i], tb = split[i], tc = ptr[i + 1];
            double2 acc = make_double2(0.0, 0.0);
            if (staged) {
                // terms inside the window: record, x and monomial all come from shared memory
#pragma unroll 4
                for (int t = ta; t < tb; ++t) {
                    const MvTerm a = mv_load_shared(srec, t);
                    const double2 xv = xs[a.col_off * 32], mv = ms[a.mono * 32];
                    acc.x = fma(a.val * mv.x, xv.x, acc.x);
                    acc.y = fma(a.val * mv.y, xv.y, acc.y);
                }
                for (int t = tb; t < tc; ++t) {
                    const MvTerm a = mv_load_shared(srec, t);
                    const double2 xv = *reinterpret_cast<const double2*>(xg + a.col_off), mv = ms[a.mono * 32];
                    acc.x = fma(a.val * mv.x, xv.x, acc.x);
                    acc.y = fma(a.val * mv.y, xv.y, acc.y);
                }
            } else {
                for (int t = ta; t < tb; ++t) {
                    const MvTerm a = mv_load(grec, t);
                    const double2 xv = xs[a.col_off * 32], mv = ms[a.mono * 32];
                    acc.x = fma(a.val * mv.x, xv.x, acc.x);
                    acc.y = fma(a.val * mv.y, xv.y, acc.y);
                }
                for (int t = tb; t < tc; ++t) {
                    const MvTerm a = mv_load(grec, t);
                    const double2 xv = *reinterpret_cast<const double2*>(xg + a.col_off), mv = ms[a.mono * 32];
                    acc.x = fma(a.val * mv.x, xv.x, acc.x);
                    acc.y = fma(a.val * mv.y, xv.y, acc.y);
                }
            }
            *reinterpret_cast<double2*>(y + (int64_t)i * DB_TILE) = acc;
        }
    }
}

extern "C" int db_batches_matvec(const db_batch* batches, int32_t nbatch, int32_t total_blocks, int32_t x_slot, int32_t ym_slot, int32_t yl_slot, void* stream)
{
    if (nbatch <= 0 || total_blocks <= 0) return 0;
#ifndef DB_EMU
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(k_batches_matvec, cudaFuncAttributeMaxDynamicSharedMemorySize, DB_MAX_SMEM);
        cudaFuncSetAttribute(k_batches_matvec, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
        attr = true;
    }
#endif
    DB_LAUNCH(k_batches_matvec, dim3(total_blocks), dim3(MV_THREADS), MV_SMEM_BYTES, stream, batches, nbatch, x_slot, ym_slot, yl_slot);
    return db_check_launch("batches_matvec");
}

// 64 x 64 tiles: one side is a full 512-byte row of the tile-major pencil vectors (64 systems), the other a 512-byte
// run of a z line; 16 independent loads per thread keep enough bytes in flight for a pure data-movement kernel.  One CTA
// owns (line kind, 64 systems) and walks the whole line in 64-element steps, so the descriptor / batch look-up in front of
// the copies is paid once per line instead of once per tile (one tile per CTA makes the kernel issue-bound).
#define MOVE_T 64
template <bool GATHER>
__global__ void __launch_bounds__(MOVE_T * 4)
k_batches_move(const db_batch* __restrict__ batches, int nbatch, int side, int slot, double* __restrict__ arena)
{
    DB_SMEM(double, tile);                         // [MOVE_T][MOVE_T + 1]
    const int bi = find_batch(batches, nbatch, blockIdx.x, 2 + side);
    const db_batch& B = batches[bi];
    const int local = blockIdx.x - B.blk_move[side];
    const int ptiles = (B.S + MOVE_T - 1) / MOVE_T;
    const int sblocks = ptiles * B.nrhs;                       // (member, pencil tile) pairs per line
    const int q = local / sblocks;
    const int mt = local - q * sblocks;
    const int member = mt / ptiles;
    const int s0 = (mt - member * ptiles) * MOVE_T;
    const int32_t* __restrict__ lp = B.line_ptr[side];
    const int lq = lp[q];
    const int len = lp[q + 1] - lq;
    const int S = B.S, ld = B.ld;
    const int64_t base = B.line_base[side][member * B.nlines[side] + q];
    const double sgn = B.line_sign[side][member * B.nlines[side] + q];   // +-1: D2 (variables) / D1 (equations) of this member
    const int64_t* __restrict__ so = B.sys_off[side] + (int64_t)B.line_kind[side][q] * ld;
    const int32_t* __restrict__ pos = B.line_pos[side] + lq;
    double* __restrict__ vec = B.vec[slot];
    const int tx = threadIdx.x, ty = threadIdx.y;
    constexpr int P = MOVE_T + 1;
    const int s = s0 + tx;                                     // system on the tile-major side
    const bool s_ok = s < S;
    double* __restrict__ vcol = vec + db_tbase(member * ld + (s_ok ? s : 0), B.n);
    // arena row bases of the (up to) 16 systems this thread touches on the line side
    int64_t rowb[MOVE_T / 4];
#pragma unroll
    for (int i = 0; i < MOVE_T / 4; ++i) {
        const int sr = s0 + ty + 4 * i;
        rowb[i] = (sr < S) ? base + so[sr] : -1;
    }
    for (int m0 = 0; m0 < len; m0 += MOVE_T) {
        if (m0 > 0) __syncthreads();                           // previous tile fully consumed
        if (GATHER) {
#pragma unroll
            for (int i = 0; i < MOVE_T / 4; ++i) {
                const int m = m0 + tx;
                if (rowb[i] >= 0 && m < len) tile[(ty + 4 * i) * P + tx] = DB_LDCS(arena + rowb[i] + m);
            }
            __syncthreads();
#pragma unroll 4
            for (int r = ty; r < MOVE_T; r += 4) {
                const int m = m0 + r;
                if (s_ok && m < len) vcol[(int64_t)pos[m] * DB_TILE] = sgn * tile[tx * P + r];
            }
        } else {
#pragma unroll 4
            for (int r = ty; r < MOVE_T; r += 4) {
                const int m = m0 + r;
                if (s_ok && m < len) tile[tx * P + r] = sgn * DB_LDCS(vcol + (int64_t)pos[m] * DB_TILE);
            }
            __syncthreads();
#pragma unroll
            for (int i = 0; i < MOVE_T / 4; ++i) {
                const int m = m0 + tx;
                if (rowb[i] >= 0 && m < len) arena[rowb[i] + m] = tile[(ty + 4 * i) * P + tx];
            }
        }
    }
}

extern "C" int db_batches_move(const db_batch* batches, int32_t nbatch, int32_t total_blocks, int32_t side, int32_t gather,
                               int32_t slot, double* arena, void* stream)
{
    if (nbatch <= 0 || total_blocks <= 0) return 0;
    if (side < 0 || side > 1 || slot < 0 || slot >= DB_MAX_VECS) { db_set_error("batches_move: bad arguments"); return 1; }
    const size_t smem = (size_t)MOVE_T * (MOVE_T + 1) * sizeof(double);
    if (gather) DB_LAUNCH(k_batches_move<true>, dim3(total_blocks), dim3(MOVE_T, 4), smem, stream, batches, nbatch, side, slot, arena);
    else DB_LAUNCH(k_batches_move<false>, dim3(total_blocks), dim3(MOVE_T, 4), smem, stream, batches, nbatch, side, slot, arena);
    return db_check_launch("batches_move");
}

__global__ void __launch_bounds__(PB_THREADS)
k_batches_assemble(const db_batch* __restrict__ batches, int nbatch, int lu_slot)
{
    const int bi = find_batch(batches, nbatch, blockIdx.x, 4);
    const db_batch& B = batches[bi];
    const int local = blockIdx.x - B.blk_assemble;
    const int sblocks = (B.S + PB_THREADS - 1) / PB_THREADS;
    const int s = (local % sblocks) * PB_THREADS + threadIdx.x;
    if (s >= B.S) return;
    const int e0 = (local / sblocks) * ASM_ENTRIES_PER_BLOCK;
    const int e1 = (e0 + ASM_ENTRIES_PER_BLOCK < B.n_entries) ? e0 + ASM_ENTRIES_PER_BLOCK : B.n_entries;
    double* __restrict__ lu = B.lu[lu_slot] + db_tbase(s, B.n_entries);
    const double* __restrict__ mono = B.mono + s;
    const int ld = B.ld;
    for (int e = e0; e < e1; ++e) {
        double v = 0.0;
        for (int t = B.asm_ptr[e]; t < B.asm_ptr[e + 1]; ++t)
            v = fma(B.asm_val[t], mono[(int64_t)B.asm_mono[t] * ld], v);
        lu[(int64_t)e * DB_TILE] = v;
    }
}

extern "C" int db_batches_assemble(const db_batch* batches, int32_t nbatch, int32_t total_blocks, int32_t lu_slot, void* stream)
{
    if (nbatch <= 0 || total_blocks <= 0) return 0;
    DB_LAUNCH(k_batches_assemble, dim3(total_blocks), dim3(PB_THREADS), 0, stream, batches, nbatch, lu_slot);
    return db_check_launch("batches_assemble");
}

// factorisation shares the solve's block map (one thread per system, SOLVE_THREADS per block)
__global__ void __launch_bounds__(SOLVE_THREADS)
k_batches_factor(const db_batch* __restrict__ batches, int nbatch, int lu_slot)
{
    const int bi = find_batch(batches, nbatch, blockIdx.x, 0);
    const db_batch& B = batches[bi];
    const int s = (blockIdx.x - B.blk_solve) * SOLVE_THREADS + threadIdx.x;
    if (s >= B.S) return;
    const int n = B.n;
    double* __restrict__ lu = B.lu[lu_slot] + db_tbase(s, B.n_entries);
    int64_t dp = 0;
    bool bad = false;
    for (int k = 0; k < n; ++k) {
        const int64_t d = (int64_t)B.diag_eid[k] * DB_TILE;
        const double piv = lu[d];
        if (!(fabs(piv) > 0.0) || !(fabs(piv) < 1e300)) bad = true;
        const double inv = 1.0 / piv;
        lu[d] = inv;
        const int u0 = B.fu_ptr[k], u1 = B.fu_ptr[k + 1];
        for (int a = B.fl_ptr[k]; a < B.fl_ptr[k + 1]; ++a) {
            const int64_t le = (int64_t)B.fl_eid[a] * DB_TILE;
            const double l = lu[le] * inv;
            lu[le] = l;
            for (int b = u0; b < u1; ++b, ++dp) {
                const int64_t de = (int64_t)B.fd_eid[dp] * DB_TILE;
                lu[de] = fma(-l, lu[(int64_t)B.fu_eid[b] * DB_TILE], lu[de]);
            }
        }
    }
    if (bad) atomicAdd(B.info, 1);
}

extern "C" int db_batches_factor(const db_batch* batches, int32_t nbatch, int32_t total_blocks, int32_t lu_slot, void* stream)
{
    if (nbatch <= 0 || total_blocks <= 0) return 0;
    DB_LAUNCH(k_batches_factor, dim3(total_blocks), dim3(SOLVE_THREADS), 0, stream, batches, nbatch, lu_slot);
    return db_check_launch("batches_factor");
}

// ---------------------------------------------------------------------------------------------------------
// Verification of a factorisation (no reference counterpart: SuperLU pivots every pencil separately,
// libraries/matsolvers.py:179-183; a pivot order shared by a batch has to be CHECKED for every member).  After
// x = LU^{-1} b (db_batches_solve) and Mx, Lx (db_batches_matvec) of a probe right-hand side b:
//     out[system] = max_i |a0 (Mx)_i + b0 (Lx)_i - b_i| / (max_i |b_i| + max_i |a0 (Mx)_i| + max_i |b0 (Lx)_i|)
// i.e. the normwise backward error of the solve (worst member of the pencil); non-finite values give +inf.  One thread per pencil (coalesced
// rows), same block map as the solve.  out has total_blocks * 64 entries (padding lanes: 0).
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SOLVE_THREADS)
k_batches_residual(const db_batch* __restrict__ batches, int nbatch, int b_slot, int m_slot, int l_slot, double a0, double b0,
                   double* __restrict__ out)
{
    const int bi = find_batch(batches, nbatch, blockIdx.x, 0);
    const db_batch& B = batches[bi];
    const int s = (blockIdx.x - B.blk_solve) * SOLVE_THREADS + threadIdx.x;
    double res = 0.0;
    if (s < B.S) {
        for (int member = 0; member < B.nrhs; ++member) {
            const int64_t tb = db_tbase(member * B.ld + s, B.n);
            const double* __restrict__ b = B.vec[b_slot] + tb;
            const double* __restrict__ m = B.vec[m_slot] + tb;
            const double* __restrict__ l = B.vec[l_slot] + tb;
            double rmax = 0.0, bmax = 0.0, mmax = 0.0, lmax = 0.0;
            bool finite = true;
            for (int i = 0; i < B.n; ++i) {
                const double bv = b[(int64_t)i * DB_TILE], mv = a0 * m[(int64_t)i * DB_TILE], lv = b0 * l[(int64_t)i * DB_TILE];
                const double r = (mv + lv) - bv;
                if (!(fabs(r) < 1e300)) finite = false;
                rmax = fmax(rmax, fabs(r)); bmax = fmax(bmax, fabs(bv)); mmax = fmax(mmax, fabs(mv)); lmax = fmax(lmax, fabs(lv));
            }
            const double den = bmax + mmax + lmax;
            res = fmax(res, !finite ? 1e300 * 1e300 : (den > 0.0 ? rmax / den : 0.0));
        }
    }
    out[(int64_t)blockIdx.x * SOLVE_THREADS + threadIdx.x] = res;
}

extern "C" int db_batches_residual(const db_batch* batches, int32_t nbatch, int32_t total_blocks, int32_t b_slot, int32_t m_slot,
                                   int32_t l_slot, double a0, double b0, double* out, void* stream)
{
    if (nbatch <= 0 || total_blocks <= 0) return 0;
    if (b_slot < 0 || m_slot < 0 || l_slot < 0 || b_slot >= DB_MAX_VECS || m_slot >= DB_MAX_VECS || l_slot >= DB_MAX_VECS) {
        db_set_error("batches_residual: bad slots"); return 1;
    }
    DB_LAUNCH(k_batches_residual, dim3(total_blocks), dim3(SOLVE_THREADS), 0, stream, batches, nbatch, b_slot, m_slot, l_slot, a0, b0, out);
    return db_check_launch("batches_residual");
}
