// Ragged batches of banded systems with partial pivoting, one warp per system (curvilinear pencil path: one system per
// azimuthal wavenumber m, coupled along the degree l; reference core/subsystems.py:497-602 builds them one by one and
// libraries/matsolvers.py:126-183 SuperLU-factors each).  Storage is LAPACK's general-band layout, column-major:
//   operator storage  (ld0 = kl + ku + 1):      A(i, j) at  ab0[(ku + i - j) + j * ld0]
//   factor storage    (ldf = 2 kl + ku + 1):    A(i, j) at  ab [(kl + ku + i - j) + j * ldf]   (kl extra rows of fill-in)
// and the elimination is the unblocked band LU with row interchanges (the algorithm of LAPACK's dgbtf2 / dgbtrs), restated
// for a warp: pivot search = shuffle arg-max over the kl + 1 candidates, interchange and rank-1 update = lanes over the
// (kl) x (ku + kl) window.  Vectors of system s: element (i, r) at vec_off + i * nrhs + r.
#include "db_common.cuh"

#ifdef DB_EMU
#define DB_WARP_SYNC() emu_yield()
#else
#define DB_WARP_SYNC() __syncwarp()
#endif

__device__ __forceinline__ int bd_min(int a, int b) { return a < b ? a : b; }
__device__ __forceinline__ int bd_max(int a, int b) { return a > b ? a : b; }
__device__ __forceinline__ bool bd_finite(double v) { return v - v == 0.0; }

#ifdef DB_EMU
#define BD_LDCG(p) (*(p))
#define BD_FENCE() ((void)0)
#else
#define BD_LDCG(p) __ldcg(p)
#define BD_FENCE() __threadfence_block()
#endif
#define BD_WARPS 4            // systems per CTA in the factor / elementwise kernels

// ---------------------------------------------------------------------------------------------------------
// LHS assembly: ab(factor storage) = a0 * M(operator storage) + b0 * L(operator storage), fill-in rows zero
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_banded_combine(const db_banded_sys* __restrict__ sys, int kl, int ku, double a0, const double* __restrict__ m_ab,
                 double b0, const double* __restrict__ l_ab, double* __restrict__ out)
{
    const db_banded_sys S = sys[blockIdx.x];
    const int ld0 = kl + ku + 1, ldf = 2 * kl + ku + 1;
    const int64_t total = (int64_t)S.n * ldf;
    for (int64_t e = (int64_t)blockIdx.y * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.y * blockDim.x) {
        const int64_t j = e / ldf; const int r = (int)(e - j * ldf);
        double v = 0.0;
        if (r >= kl) {
            const int64_t src = S.op_off + j * ld0 + (r - kl);
            v = a0 * m_ab[src] + b0 * l_ab[src];
        }
        out[S.lu_off + e] = v;
    }
}

extern "C" int db_banded_combine(const db_banded_sys* sys, int32_t nsys, int32_t kl, int32_t ku, double a0, const double* m_ab,
                                 double b0, const double* l_ab, double* out, void* stream)
{
    if (nsys <= 0) return 0;
    DB_LAUNCH(k_banded_combine, dim3((unsigned)nsys, 8), dim3(256), 0, stream, sys, kl, ku, a0, m_ab, b0, l_ab, out);
    return db_check_launch("banded_combine");
}

// ---------------------------------------------------------------------------------------------------------
// Factorisation: P A = L U in place (band LU with partial pivoting), one warp per system.
// info[s] = number of exactly-zero / non-finite pivots met (0 = ok)
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32 * BD_WARPS)
k_banded_factor(const db_banded_sys* __restrict__ sys, int nsys, int kl, int ku, double* ab_all,
                int32_t* __restrict__ ipiv_all, int32_t* __restrict__ info)
{
    const int lane = threadIdx.x & 31;
    const int s = blockIdx.x * BD_WARPS + (threadIdx.x >> 5);
    // all warps of the CTA keep running to the end (no early return: the emulated scheduler steps every fiber)
    const bool live = s < nsys;
    const db_banded_sys S = sys[live ? s : 0];
    const int n = live ? S.n : 0;
    const int kv = kl + ku, ldf = 2 * kl + ku + 1;
    double* ab = ab_all + S.lu_off;
    int32_t* __restrict__ ipiv = ipiv_all + S.piv_off;
    int ju = 0, bad = 0;
    // band entries that other lanes wrote are re-read from L2 (ld.global.cg) behind a CTA fence, not through the SM's L1
#define BD_SYNC() do { BD_FENCE(); DB_WARP_SYNC(); } while (0)
    for (int j = 0; j < n; ++j) {
        const int km = bd_min(kl, n - 1 - j);
        double* colj = ab + (int64_t)j * ldf + kv;                       // colj[l] = A(j + l, j)
        // pivot search: largest |A(j + l, j)|, l = 0 .. km, lowest l on ties
        double best = -1.0; int bl = 0;
        for (int l = lane; l <= km; l += 32) {
            const double v = fabs(BD_LDCG(colj + l));
            if (v > best) { best = v; bl = l; }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const double ob = __shfl_down_sync(0xffffffffu, best, off);
            const int ol = (int)__shfl_down_sync(0xffffffffu, (double)bl, off);
            if (ob > best || (ob == best && ol < bl)) { best = ob; bl = ol; }
        }
        best = __shfl_sync(0xffffffffu, best, 0);
        const int jp = (int)__shfl_sync(0xffffffffu, (double)bl, 0);
        if (lane == 0) ipiv[j] = j + jp;
        if (!(best > 0.0) || !bd_finite(best)) { ++bad; continue; }
        ju = bd_max(ju, bd_min(j + ku + jp, n - 1));
        // interchange rows j and j + jp over columns j .. ju:  A(r, c) at ab[kv + r - c + c * ldf]
        if (jp != 0) {
            for (int c = j + lane; c <= ju; c += 32) {
                double* p = ab + (int64_t)c * ldf + kv + (j - c);
                const double t = BD_LDCG(p), u = BD_LDCG(p + jp); p[0] = u; p[jp] = t;
            }
        }
        BD_SYNC();
        const double rp = 1.0 / BD_LDCG(colj);
        BD_SYNC();
        for (int l = 1 + lane; l <= km; l += 32) colj[l] = BD_LDCG(colj + l) * rp;
        BD_SYNC();
        // trailing update A(j + l, c) -= L(l) * U(j, c),  l = 1 .. km,  c = j + 1 .. ju
        const int nc = ju - j;
        for (int idx = lane; idx < nc * km; idx += 32) {
            const int cc = idx / km, l = 1 + idx - cc * km;
            const int c = j + 1 + cc;
            double* p = ab + (int64_t)c * ldf + kv + (j - c);             // p[0] = U(j, c), p[l] = A(j + l, c)
            p[l] = fma(-BD_LDCG(colj + l), BD_LDCG(p), BD_LDCG(p + l));
        }
        BD_SYNC();
    }
#undef BD_SYNC
    if (live && lane == 0) info[s] = bad;
}

extern "C" int db_banded_factor(const db_banded_sys* sys, int32_t nsys, int32_t kl, int32_t ku, double* ab, int32_t* ipiv,
                                int32_t* info, void* stream)
{
    if (nsys <= 0) return 0;
    DB_LAUNCH(k_banded_factor, dim3((unsigned)((nsys + BD_WARPS - 1) / BD_WARPS)), dim3(32 * BD_WARPS), 0, stream,
              sys, nsys, kl, ku, ab, ipiv, info);
    return db_check_launch("banded_factor");
}

// ---------------------------------------------------------------------------------------------------------
// Solve  x = A^{-1} (sum_k coef_k v_k)  for every right-hand-side column, both triangular sweeps in one launch.
// CTA = one warp = one (system, chunk of RC columns).  The right-hand side (combined on the fly from up to 16 vectors: the
// IMEX stage combination of core/timesteppers.py:617-623) is staged ONCE in shared memory, both sweeps run there, and the
// factor columns are read straight from global memory.
// ---------------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(32)
k_banded_solve(const db_banded_sys* __restrict__ sys, int kl, int ku, const double* __restrict__ ab_all,
               const int32_t* __restrict__ ipiv_all, db_veccomb rhs, double* __restrict__ x_all, int RC)
{
    DB_SMEM(double, smem);
    const db_banded_sys S = sys[blockIdx.x];
    const int lane = threadIdx.x;
    const int n = S.n, nrhs = S.nrhs;
    const int r0 = blockIdx.y * RC;
    if (r0 >= nrhs) return;
    const int R = bd_min(RC, nrhs - r0);
    const int kv = kl + ku, ldf = 2 * kl + ku + 1;
    double* __restrict__ b = smem;                                   // [n][R]
    int32_t* __restrict__ piv = reinterpret_cast<int32_t*>(smem + (int64_t)n * RC);     // [n]
    const double* __restrict__ ab = ab_all + S.lu_off;
    // stage: combined right-hand side and the pivot rows
    for (int64_t e = lane; e < (int64_t)n * R; e += 32) {
        const int64_t i = e / R; const int r = (int)(e - i * R);
        const int64_t g = S.vec_off + i * nrhs + r0 + r;
        double acc = 0.0;
        for (int k = 0; k < rhs.nvec; ++k) acc = fma(rhs.coef[k], rhs.vec[k][g], acc);
        b[i * R + r] = acc;
    }
    for (int i = lane; i < n; i += 32) piv[i] = ipiv_all[S.piv_off + i] - i;
    // ---- forward sweep: y = L^{-1} P b
    DB_WARP_SYNC();
    for (int j = 0; j < n; ++j) {
        const int km = bd_min(kl, n - 1 - j);
        const int p = piv[j];
        if (p != 0) {
            for (int r = lane; r < R; r += 32) { const double t = b[j * R + r]; b[j * R + r] = b[(j + p) * R + r]; b[(j + p) * R + r] = t; }
            DB_WARP_SYNC();
        }
        const double* col = ab + (int64_t)j * ldf + kv;
        for (int idx = lane; idx < km * R; idx += 32) {
            const int l = 1 + idx / R, r = idx % R;
            b[(j + l) * R + r] = fma(-col[l], b[j * R + r], b[(j + l) * R + r]);
        }
        DB_WARP_SYNC();
    }
    // ---- backward sweep: x = U^{-1} y  (column oriented: x_j = y_j / U_jj, then y_i -= U_ij x_j for i = j - kv .. j - 1)
    for (int j = n - 1; j >= 0; --j) {
        const double* col = ab + (int64_t)j * ldf + kv;                  // col[i - j] = U(i, j), i <= j
        const double rd = 1.0 / col[0];
        for (int r = lane; r < R; r += 32) b[j * R + r] *= rd;
        DB_WARP_SYNC();
        const int ku2 = bd_min(kv, j);
        for (int idx = lane; idx < ku2 * R; idx += 32) {
            const int l = 1 + idx / R, r = idx % R;
            b[(j - l) * R + r] = fma(-col[-l], b[j * R + r], b[(j - l) * R + r]);
        }
        DB_WARP_SYNC();
    }
    for (int64_t e = lane; e < (int64_t)n * R; e += 32) {
        const int64_t i = e / R; const int r = (int)(e - i * R);
        x_all[S.vec_off + i * nrhs + r0 + r] = b[i * R + r];
    }
}

extern "C" int db_banded_solve(const db_banded_sys* sys, int32_t nsys, int32_t kl, int32_t ku, int32_t max_n, int32_t max_nrhs,
                               const double* ab, const int32_t* ipiv, const db_veccomb* rhs, double* x, void* stream)
{
    if (nsys <= 0 || max_n <= 0 || max_nrhs <= 0) return 0;
    if (rhs->nvec < 1 || rhs->nvec > 16) { db_set_error("banded_solve: 1..16 right-hand-side vectors"); return 1; }
    // columns per CTA: as many as fit 96 KB (the sweeps of different chunks are independent)
    int RC = max_nrhs < 8 ? max_nrhs : 8;
    while (RC > 1 && (size_t)max_n * RC * 8 > 96 * 1024) RC >>= 1;
    const size_t smem = (size_t)max_n * RC * sizeof(double) + (size_t)max_n * sizeof(int32_t);
    if (smem > DB_MAX_SMEM) { db_set_error("banded_solve: system of size %d does not fit shared memory", max_n); return 1; }
    static bool attr_set = false;
    if (!attr_set) { DB_SET_SMEM_ATTR(k_banded_solve); attr_set = true; }
    DB_LAUNCH(k_banded_solve, dim3((unsigned)nsys, (unsigned)((max_nrhs + RC - 1) / RC)), dim3(32), smem, stream,
              sys, kl, ku, ab, ipiv, *rhs, x, RC);
    return db_check_launch("banded_solve");
}

// ---------------------------------------------------------------------------------------------------------
// y = A x for up to two band operators at once (M.X and L.X of core/timesteppers.py:590-591, 604); operator storage.
// One thread per (row, column of right-hand sides).
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_banded_matvec(const db_banded_sys* __restrict__ sys, int kl, int ku, const double* __restrict__ a_ab, const double* __restrict__ b_ab,
                const double* __restrict__ x, double* __restrict__ ya, double* __restrict__ yb)
{
    const db_banded_sys S = sys[blockIdx.x];
    const int ld0 = kl + ku + 1;
    const int64_t total = (int64_t)S.n * S.nrhs;
    for (int64_t e = (int64_t)blockIdx.y * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.y * blockDim.x) {
        const int i = (int)(e / S.nrhs); const int r = (int)(e - (int64_t)i * S.nrhs);
        const int c0 = bd_max(0, i - kl), c1 = bd_min(S.n - 1, i + ku);
        double sa = 0.0, sb = 0.0;
        for (int c = c0; c <= c1; ++c) {
            const int64_t a = S.op_off + (int64_t)c * ld0 + (ku + i - c);
            const double xv = x[S.vec_off + (int64_t)c * S.nrhs + r];
            if (ya) sa = fma(a_ab[a], xv, sa);
            if (yb) sb = fma(b_ab[a], xv, sb);
        }
        if (ya) ya[S.vec_off + e] = sa;
        if (yb) yb[S.vec_off + e] = sb;
    }
}

extern "C" int db_banded_matvec(const db_banded_sys* sys, int32_t nsys, int32_t kl, int32_t ku, const double* a_ab, const double* b_ab,
                                const double* x, double* ya, double* yb, void* stream)
{
    if (nsys <= 0) return 0;
    DB_LAUNCH(k_banded_matvec, dim3((unsigned)nsys, 8), dim3(256), 0, stream, sys, kl, ku, a_ab, b_ab, x, ya, yb);
    return db_check_launch("banded_matvec");
}

// ---------------------------------------------------------------------------------------------------------
// Gather / scatter between a coefficient arena and pencil vectors through an index table (S2):
//   gather : vec[e] = idx[e] >= 0 ? arena[idx[e]] : 0        scatter: arena[idx[e]] = vec[e] where idx[e] >= 0
// (invalid modes -- l < bd_max(|m|, |s|), the -sin part of l = 0 -- carry identity rows, core/basis.py:3178-3211)
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_index_move(const int64_t* __restrict__ idx, int64_t count, double* __restrict__ arena, double* __restrict__ vec, int gather)
{
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < count; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t a = idx[e];
        if (gather) vec[e] = a >= 0 ? arena[a] : 0.0;
        else if (a >= 0) arena[a] = vec[e];
    }
}

extern "C" int db_index_move(const int64_t* idx, int64_t count, double* arena, double* vec, int32_t gather, void* stream)
{
    if (count <= 0) return 0;
    int64_t blocks = (count + 255) / 256;
    if (blocks > (int64_t)db_num_sms() * 8) blocks = (int64_t)db_num_sms() * 8;
    DB_LAUNCH(k_index_move, dim3((unsigned)blocks), dim3(256), 0, stream, idx, count, arena, vec, gather);
    return db_check_launch("index_move");
}

// the same for contiguous RUNS of `run` doubles per index entry (row permutations of the curvilinear transposes: one entry per
// coefficient row): gather: vec[e * run + x] = arena[idx[e] + x];  scatter: arena[idx[e] + x] = vec[e * run + x]
__global__ void __launch_bounds__(256)
k_index_move_runs(const int64_t* __restrict__ idx, int64_t run, double* __restrict__ arena, double* __restrict__ vec, int gather)
{
    const int64_t e = blockIdx.x;
    const int64_t a = idx[e];
    if (a < 0) {
        if (gather) for (int64_t x = (int64_t)blockIdx.y * blockDim.x + threadIdx.x; x < run; x += (int64_t)gridDim.y * blockDim.x) vec[e * run + x] = 0.0;
        return;
    }
    for (int64_t x = (int64_t)blockIdx.y * blockDim.x + threadIdx.x; x < run; x += (int64_t)gridDim.y * blockDim.x) {
        if (gather) vec[e * run + x] = arena[a + x];
        else arena[a + x] = vec[e * run + x];
    }
}

extern "C" int db_index_move_runs(const int64_t* idx, int64_t count, int64_t run, double* arena, double* vec, int32_t gather, void* stream)
{
    if (count <= 0 || run <= 0) return 0;
    if (count > 2147483647LL) { db_set_error("index_move_runs: too many entries"); return 1; }
    int yb = (int)((run + 255) / 256);
    if (yb > 64) yb = 64;
    DB_LAUNCH(k_index_move_runs, dim3((unsigned)count, (unsigned)yb), dim3(256), 0, stream, idx, run, arena, vec, gather);
    return db_check_launch("index_move_runs");
}

// ---------------------------------------------------------------------------------------------------------
// Complex linear combinations on (cos, -sin) pairs: arrays (ncomp, 2 * npair, ncol), a pair = two adjacent rows holding the
// real and imaginary part of the coefficient of exp(i m phi) (core/basis.py:1108-1134).  For output component o
//     out[o] = sum_{t in terms of o} (re_t + i im_t) * in[src_t]
// where re_t / im_t are constants, optionally times a per-element symbol: syms[sym_off + (j * ncol + c) / sym_div] (sym_off >= 0;
// sym_div > 1 when the symbol does not depend on the trailing sym_div entries of a row, e.g. the radial index of shell data).
// Serves (a) the separable sphere operators in coefficient space -- gradient, divergence, Laplacian, skew: symbols
// k(l, s, mu) per degree, core/basis.py:3299-3420, core/operators.py:2125-2160 -- and (b) the component <-> spin
// recombination in (azimuthal coefficient, colatitude grid) space (libraries/spin_recombination.pyx:9-56,
// core/coords.py:219-232).
// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_pair_lincomb(const double* __restrict__ in, double* __restrict__ out, int64_t npair, int64_t ncol, int n_out,
               const int32_t* __restrict__ term_ptr, const db_pair_lin_term* __restrict__ terms, const double* __restrict__ syms,
               int64_t sym_div)
{
    const int64_t plane = 2 * npair * ncol;
    const int64_t total = npair * ncol;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t j = e / ncol, c = e - j * ncol;
        const int64_t o_re = (2 * j) * ncol + c, o_im = o_re + ncol;
        for (int o = 0; o < n_out; ++o) {
            double ar = 0.0, ai = 0.0;
            for (int t = term_ptr[o]; t < term_ptr[o + 1]; ++t) {
                const db_pair_lin_term T = terms[t];
                double sr = T.re, si = T.im;
                if (T.sym_off >= 0) { const double sv = syms[T.sym_off + e / sym_div]; sr *= sv; si *= sv; }
                const double xr = in[T.src * plane + o_re], xi = in[T.src * plane + o_im];
                ar += sr * xr - si * xi;
                ai += sr * xi + si * xr;
            }
            out[o * plane + o_re] = ar;
            out[o * plane + o_im] = ai;
        }
    }
}

extern "C" int db_pair_lincomb(const double* in, double* out, int64_t npair, int64_t ncol, int32_t n_out,
                               const int32_t* term_ptr, const db_pair_lin_term* terms, const double* syms, int64_t sym_div, void* stream)
{
    const int64_t total = npair * ncol;
    if (total <= 0 || n_out <= 0) return 0;
    if (sym_div < 1) sym_div = 1;
    int64_t blocks = (total + 255) / 256;
    if (blocks > (int64_t)db_num_sms() * 8) blocks = (int64_t)db_num_sms() * 8;
    DB_LAUNCH(k_pair_lincomb, dim3((unsigned)blocks), dim3(256), 0, stream, in, out, npair, ncol, n_out, term_ptr, terms, syms, sym_div);
    return db_check_launch("pair_lincomb");
}
