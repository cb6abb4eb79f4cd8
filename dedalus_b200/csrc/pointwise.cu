// Grid-space products (P1): generic "sum of products" evaluator and dense matrix transform (T4).
//
// Reference: DotProduct.operate (np.einsum), MultiplyFields.operate, AddFields.operate evaluated one node at a
// time on full grid arrays (core/arithmetic.py:246-251, 666-674, 855-866) -> every intermediate is a full HBM
// round trip.  Here the whole right-hand-side polynomial of an equation set is one kernel: each CTA stages a
// tile of all inputs in shared memory (every input element read from HBM exactly once, coalesced), evaluates
// all outputs from it and writes each output once.
#include "db_common.cuh"
#include <cstdlib>
#include <cstdint>

#define PW_TILE 256

// launches per kernel so far (db_pointwise_launches): k_pointwise, k_pointwise_v3, k_pointwise_pairs, transpose 16-byte branch,
// transpose 8-byte branch
static long long g_pw_launches[5] = {0, 0, 0, 0, 0};
extern "C" long long db_pointwise_launches(int32_t kind) { return kind >= 0 && kind < 5 ? g_pw_launches[kind] : -1; }

__global__ void __launch_bounds__(PW_TILE)
k_pointwise(const double* __restrict__ in, double* __restrict__ out, int64_t npoints, int n_in, int n_out,
            const int32_t* __restrict__ term_ptr, const double* __restrict__ coef,
            const int32_t* __restrict__ fac_ptr, const int32_t* __restrict__ fac)
{
    DB_SMEM(double, tile);                         // [n_in][PW_TILE]
    for (int64_t p0 = (int64_t)blockIdx.x * PW_TILE; p0 < npoints; p0 += (int64_t)gridDim.x * PW_TILE) {
        const int64_t p = p0 + threadIdx.x;
        const bool live = p < npoints;
        for (int i = 0; i < n_in; ++i)
            tile[i * PW_TILE + threadIdx.x] = live ? in[(int64_t)i * npoints + p] : 0.0;
        // each thread only touches its own column: no barrier needed
        if (live) {
            for (int o = 0; o < n_out; ++o) {
                double acc = 0.0;
                for (int t = term_ptr[o]; t < term_ptr[o + 1]; ++t) {
                    double prod = coef[t];
                    for (int f = fac_ptr[t]; f < fac_ptr[t + 1]; ++f)
                        prod *= tile[fac[f] * PW_TILE + threadIdx.x];
                    acc += prod;
                }
                out[(int64_t)o * npoints + p] = acc;
            }
        }
    }
}

// v3: two points per thread, staged with 16-byte asynchronous copies (cp.async, L1 bypass), double buffered:
// the n_in loads of the NEXT tile are in flight while the current tile's products are evaluated, and no load result
// ever sits on a register dependency.  Each thread only reads the slots it filled itself, so no block barrier.
#define PW3_T 128
__global__ void __launch_bounds__(PW3_T)
k_pointwise_v3(const double* __restrict__ in, double* __restrict__ out, int64_t npoints, int n_in, int n_out,
               const int32_t* __restrict__ term_ptr, const double* __restrict__ coef,
               const int32_t* __restrict__ fac_ptr, const int32_t* __restrict__ fac)
{
    DB_SMEM(double, tile);                         // 2 buffers of [n_in][PW3_T] double2
    double2* tile2 = reinterpret_cast<double2*>(tile);
    const int64_t np2 = npoints >> 1;
    const int64_t stride = (int64_t)gridDim.x * PW3_T;
    int64_t q = (int64_t)blockIdx.x * PW3_T + threadIdx.x;
    auto stage = [&](int64_t qq, int buf) {
        if (qq < np2) {
            double2* dst = tile2 + (size_t)buf * n_in * PW3_T + threadIdx.x;
            const double* src = in + 2 * qq;
            for (int i = 0; i < n_in; ++i) db_cp_async16(dst + i * PW3_T, src + (int64_t)i * npoints);
        }
    };
    int buf = 0;
    stage(q, 0);
    db_cp_commit();
    for (; q - threadIdx.x < np2; q += stride, buf ^= 1) {        // block-uniform trip count
        stage(q + stride, buf ^ 1);
        db_cp_commit();
        db_cp_wait<1>();
        if (q < np2) {
            const double2* mine = tile2 + (size_t)buf * n_in * PW3_T + threadIdx.x;
            for (int o = 0; o < n_out; ++o) {
                double a0 = 0.0, a1 = 0.0;
                for (int t = term_ptr[o]; t < term_ptr[o + 1]; ++t) {
                    double p0 = coef[t], p1 = p0;
                    for (int f = fac_ptr[t]; f < fac_ptr[t + 1]; ++f) {
                        const double2 v = mine[fac[f] * PW3_T];
                        p0 *= v.x; p1 *= v.y;
                    }
                    a0 += p0; a1 += p1;
                }
                DB_CHECK_ALIGN16(out + (int64_t)o * npoints + 2 * q);
                reinterpret_cast<double2*>(out + (int64_t)o * npoints)[q] = make_double2(a0, a1);
            }
        }
    }
    db_cp_wait<0>();
}

// Products of at most two fields (every quadratic right-hand side: u.grad(u), u.grad(b), ...): terms are 16-byte records
// {coef, a, b} read with one warp-uniform load, so a term costs two shared loads and four flops instead of the general
// interpreter's pointer chasing (about a thousand warp instructions per pair of points, which makes the general kernel
// bound by instruction issue).  Same double-buffered asynchronous staging as k_pointwise_v3.
struct PwPair { double coef; int a; int b; };
__device__ __forceinline__ PwPair pw_load(const db_pair_term* __restrict__ rec, int t)
{
#ifdef DB_EMU
    PwPair r; r.coef = rec[t].coef; r.a = rec[t].a; r.b = rec[t].b; return r;
#else
    const int4 raw = __ldg(reinterpret_cast<const int4*>(rec) + t);
    PwPair r; r.coef = __hiloint2double(raw.y, raw.x); r.a = raw.z; r.b = raw.w; return r;
#endif
}

__global__ void __launch_bounds__(PW3_T)
k_pointwise_pairs(const double* __restrict__ in, double* __restrict__ out, int64_t npoints, int n_in, int n_out,
                  const int32_t* __restrict__ term_ptr, const db_pair_term* __restrict__ rec)
{
    DB_SMEM(double, tile);                         // 2 buffers of [n_in][PW3_T] double2
    double2* tile2 = reinterpret_cast<double2*>(tile);
    const int64_t np2 = npoints >> 1;
    const int64_t stride = (int64_t)gridDim.x * PW3_T;
    int64_t q = (int64_t)blockIdx.x * PW3_T + threadIdx.x;
    auto stage = [&](int64_t qq, int buf) {
        if (qq < np2) {
            double2* dst = tile2 + (size_t)buf * n_in * PW3_T + threadIdx.x;
            const double* src = in + 2 * qq;
            for (int i = 0; i < n_in; ++i) db_cp_async16(dst + i * PW3_T, src + (int64_t)i * npoints);
        }
    };
    int buf = 0;
    stage(q, 0);
    db_cp_commit();
    for (; q - threadIdx.x < np2; q += stride, buf ^= 1) {        // block-uniform trip count
        stage(q + stride, buf ^ 1);
        db_cp_commit();
        db_cp_wait<1>();
        if (q < np2) {
            const double2* mine = tile2 + (size_t)buf * n_in * PW3_T + threadIdx.x;
            int t = term_ptr[0];
            for (int o = 0; o < n_out; ++o) {
                const int t1 = term_ptr[o + 1];
                double a0 = 0.0, a1 = 0.0;
                for (; t < t1; ++t) {
                    const PwPair r = pw_load(rec, t);
                    const double2 va = mine[r.a * PW3_T];
                    double p0 = r.coef * va.x, p1 = r.coef * va.y;
                    if (r.b >= 0) {
                        const double2 vb = mine[r.b * PW3_T];
                        a0 = fma(p0, vb.x, a0); a1 = fma(p1, vb.y, a1);
                    } else { a0 += p0; a1 += p1; }
                }
                DB_CHECK_ALIGN16(out + (int64_t)o * npoints + 2 * q);
                reinterpret_cast<double2*>(out + (int64_t)o * npoints)[q] = make_double2(a0, a1);
            }
        }
    }
    db_cp_wait<0>();
}

extern "C" int db_pointwise_pairs(const double* in, double* out, int64_t npoints, int32_t n_in, int32_t n_out,
                                  const int32_t* term_ptr, const db_pair_term* terms, void* stream)
{
    if (npoints <= 0 || n_out <= 0) return 0;
    const size_t smem3 = (size_t)2 * n_in * PW3_T * sizeof(double2);
    if ((npoints & 1) || ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) || smem3 > (size_t)DB_MAX_SMEM) {
        db_set_error("pointwise_pairs: needs an even point count, 16-byte aligned arrays and at most %d inputs", (int)(DB_MAX_SMEM / (2 * PW3_T * sizeof(double2))));
        return 1;
    }
    if (reinterpret_cast<uintptr_t>(terms) & 15) {         // read as int4 records
        db_set_error("pointwise_pairs: the term records must be 16-byte aligned");
        return 1;
    }
    int per_sm = (int)((size_t)(226 * 1024) / (smem3 + 1024));
    if (per_sm > 8) per_sm = 8;
    int64_t blocks = (npoints / 2 + PW3_T - 1) / PW3_T;
    if (blocks > (int64_t)db_num_sms() * per_sm) blocks = (int64_t)db_num_sms() * per_sm;
#ifndef DB_EMU
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(k_pointwise_pairs, cudaFuncAttributeMaxDynamicSharedMemorySize, DB_MAX_SMEM);
        cudaFuncSetAttribute(k_pointwise_pairs, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
        attr = true;
    }
#endif
    DB_LAUNCH(k_pointwise_pairs, dim3((unsigned)blocks), dim3(PW3_T), smem3, stream, in, out, npoints, n_in, n_out, term_ptr, terms);
    ++g_pw_launches[2];
    return db_check_launch("pointwise_pairs");
}

extern "C" int db_pointwise(const double* in, double* out, int64_t npoints, int32_t n_in, int32_t n_out,
                            const int32_t* term_ptr, const double* coef, const int32_t* fac_ptr, const int32_t* fac, int32_t nfac_total,
                            void* stream)
{
    (void)nfac_total;
    if (npoints <= 0 || n_out <= 0) return 0;
    const bool vec = (npoints % 2 == 0) && ((reinterpret_cast<uintptr_t>(in) & 15) == 0) && ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
    const size_t smem3 = (size_t)2 * n_in * PW3_T * sizeof(double2);
    if (vec && smem3 <= (size_t)DB_MAX_SMEM) {
        int per_sm = (int)((size_t)(226 * 1024) / (smem3 + 1024));
        if (per_sm > 8) per_sm = 8;
        int64_t blocks3 = (npoints / 2 + PW3_T - 1) / PW3_T;
        if (blocks3 > (int64_t)db_num_sms() * per_sm) blocks3 = (int64_t)db_num_sms() * per_sm;
#ifndef DB_EMU
        static bool attr3 = false;
        if (!attr3) {
            cudaFuncSetAttribute(k_pointwise_v3, cudaFuncAttributeMaxDynamicSharedMemorySize, DB_MAX_SMEM);
            cudaFuncSetAttribute(k_pointwise_v3, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
            attr3 = true;
        }
#endif
        DB_LAUNCH(k_pointwise_v3, dim3((unsigned)blocks3), dim3(PW3_T), smem3, stream, in, out, npoints, n_in, n_out, term_ptr, coef, fac_ptr, fac);
        ++g_pw_launches[1];
        return db_check_launch("pointwise");
    }
    // odd point count, a misaligned array, or more inputs than v3's two buffers hold: one point per thread, single buffered
    const size_t smem = (size_t)n_in * PW_TILE * sizeof(double);
    if (smem > (size_t)DB_MAX_SMEM) {
        db_set_error("pointwise: too many inputs (%d, at most %d)", n_in, (int)(DB_MAX_SMEM / (PW_TILE * sizeof(double))));
        return 1;
    }
    int64_t blocks = (npoints + PW_TILE - 1) / PW_TILE;
    const int64_t cap = (int64_t)db_num_sms() * 8;
    if (blocks > cap) blocks = cap;
#ifndef DB_EMU
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(k_pointwise, cudaFuncAttributeMaxDynamicSharedMemorySize, DB_MAX_SMEM);
        attr = true;
    }
#endif
    DB_LAUNCH(k_pointwise, dim3((unsigned)blocks), dim3(PW_TILE), smem, stream, in, out, npoints, n_in, n_out, term_ptr, coef, fac_ptr, fac);
    ++g_pw_launches[0];
    return db_check_launch("pointwise");
}

// ---------------------------------------------------------------------------------------------------------
// Dense matrix transform along an axis (T4): out(o, i, r) = sum_j mat[i][j] in(o, j, r)
// 64x64 output tiles, k-blocks of 16 staged in shared memory, 4x4 register micro-tiles (fp64 FMA pipe).
// ---------------------------------------------------------------------------------------------------------
#define MM_BM 64
#define MM_BN 64
#define MM_BK 16
__global__ void __launch_bounds__(256)
k_mmt(const double* __restrict__ mat, int m, int n, const double* __restrict__ in, double* __restrict__ out, int64_t outer, int64_t inner)
{
    DB_SMEM(double, sm);
    double* As = sm;                     // [BK][BM]   (mat tile, transposed)
    double* Bs = sm + MM_BK * MM_BM;     // [BK][BN]
    const int64_t o = blockIdx.z;
    const int i0 = blockIdx.y * MM_BM;
    const int64_t r0 = (int64_t)blockIdx.x * MM_BN;
    const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
    double acc[4][4];
    for (int a = 0; a < 4; ++a) for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
    const double* inb = in + o * n * inner;
    for (int k0 = 0; k0 < n; k0 += MM_BK) {
        for (int e = threadIdx.x; e < MM_BK * MM_BM; e += 256) {
            int kk = e % MM_BK, ii = e / MM_BK;
            int gi = i0 + ii, gk = k0 + kk;
            As[kk * MM_BM + ii] = (gi < m && gk < n) ? mat[(int64_t)gi * n + gk] : 0.0;
        }
        for (int e = threadIdx.x; e < MM_BK * MM_BN; e += 256) {
            int rr = e % MM_BN, kk = e / MM_BN;
            int64_t gr = r0 + rr; int gk = k0 + kk;
            Bs[kk * MM_BN + rr] = (gr < inner && gk < n) ? inb[(int64_t)gk * inner + gr] : 0.0;
        }
        __syncthreads();
        for (int kk = 0; kk < MM_BK; ++kk) {
            double av[4], bv[4];
            for (int a = 0; a < 4; ++a) av[a] = As[kk * MM_BM + ty * 4 + a];
            for (int b = 0; b < 4; ++b) bv[b] = Bs[kk * MM_BN + tx * 4 + b];
            for (int a = 0; a < 4; ++a) for (int b = 0; b < 4; ++b) acc[a][b] = fma(av[a], bv[b], acc[a][b]);
        }
        __syncthreads();
    }
    double* outb = out + o * m * inner;
    for (int a = 0; a < 4; ++a) {
        int gi = i0 + ty * 4 + a;
        if (gi >= m) continue;
        for (int b = 0; b < 4; ++b) {
            int64_t gr = r0 + tx * 4 + b;
            if (gr < inner) outb[(int64_t)gi * inner + gr] = acc[a][b];
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// The same contraction on the FP64 tensor cores (DMMA.8x8x4 via mma.sync.m8n8k4.f64: wgmma has no FP64 path, so this is the
// tensor pipe for double precision on sm_90a).  CTA tile 64 (rows of mat) x 64 (inner), 4 warps of 32 x 32 = 4 x 4 DMMA
// tiles each (32 accumulator registers per thread); k in blocks of 16, double-buffered with 16-byte cp.async (LDGSTS,
// zero-filled outside the matrix), shared-memory rows padded (+4 doubles) so that both fragment loads are conflict-free:
//   A fragment: lane t holds mat[m0 + t/4][k + t%4]       -> As[row][k], row stride 20 doubles
//   B fragment: lane t holds in[k + t%4][r0 + t/4]        -> Bs[k][col], row stride 68 doubles
//   C fragment: lane t holds out[m0 + t/4][r0 + 2 (t%4) + {0, 1}]
// Requirements of this path: n and inner even, 16-byte aligned pointers (else the FMA-pipe kernel above runs).
// ---------------------------------------------------------------------------------------------------------
#define DM_BM 64
#define DM_BN 64
#define DM_BK 16
#define DM_AS (DM_BK + 4)
#define DM_BS (DM_BN + 4)
__global__ void __launch_bounds__(128)
k_mmt_dmma(const double* __restrict__ mat, int m, int n, const double* __restrict__ in, double* __restrict__ out, int64_t inner)
{
    DB_SHARED_ARRAY(double, As, [2][DM_BM * DM_AS]);
    DB_SHARED_ARRAY(double, Bs, [2][DM_BK * DM_BS]);
    const int64_t o = blockIdx.z;
    const int i0 = blockIdx.y * DM_BM;
    const int64_t r0 = (int64_t)blockIdx.x * DM_BN;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;
    const double* __restrict__ inb = in + o * (int64_t)n * inner;
    auto stage = [&](int buf, int k0) {
        // A: 64 rows x 8 chunks of 2 doubles;  B: 16 rows x 32 chunks
#pragma unroll
        for (int e = tid; e < DM_BM * (DM_BK / 2); e += 128) {
            const int row = e >> 3, c = e & 7;
            const int gi = i0 + row, gk = k0 + 2 * c;
            const bool ok = gi < m && gk < n;
            db_cp_async16_zfill(&As[buf][row * DM_AS + 2 * c], ok ? mat + (int64_t)gi * n + gk : mat, ok);
        }
#pragma unroll
        for (int e = tid; e < DM_BK * (DM_BN / 2); e += 128) {
            const int kk = e >> 5, c = e & 31;
            const int gk = k0 + kk; const int64_t gr = r0 + 2 * c;
            const bool ok = gk < n && gr < inner;
            db_cp_async16_zfill(&Bs[buf][kk * DM_BS + 2 * c], ok ? inb + (int64_t)gk * inner + gr : inb, ok);
        }
        db_cp_commit();
    };
    double acc[4][4][2];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) { acc[a][b][0] = 0.0; acc[a][b][1] = 0.0; }
    const int nk = (n + DM_BK - 1) / DM_BK;
    stage(0, 0);
    for (int kb = 0; kb < nk; ++kb) {
        const int buf = kb & 1;
        if (kb + 1 < nk) { stage(buf ^ 1, (kb + 1) * DM_BK); db_cp_wait<1>(); } else db_cp_wait<0>();
        __syncthreads();
        const double* __restrict__ A = As[buf] + (wm + (lane >> 2)) * DM_AS + (lane & 3);
        const double* __restrict__ B = Bs[buf] + (lane & 3) * DM_BS + wn + (lane >> 2);
#pragma unroll
        for (int k4 = 0; k4 < DM_BK; k4 += 4) {
            double af[4], bf[4];
#pragma unroll
            for (int a = 0; a < 4; ++a) af[a] = A[a * 8 * DM_AS + k4];
#pragma unroll
            for (int b = 0; b < 4; ++b) bf[b] = B[k4 * DM_BS + b * 8];
#pragma unroll
            for (int a = 0; a < 4; ++a)
#pragma unroll
                for (int b = 0; b < 4; ++b)
                    db_dmma_m8n8k4(acc[a][b][0], acc[a][b][1], af[a], bf[b]);
        }
        __syncthreads();
    }
    double* outb = out + o * (int64_t)m * inner;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
        const int gi = i0 + wm + a * 8 + (lane >> 2);
        if (gi >= m) continue;
#pragma unroll
        for (int b = 0; b < 4; ++b) {
            const int64_t gr = r0 + wn + b * 8 + 2 * (lane & 3);
            if (gr < inner) {
                DB_CHECK_ALIGN16(outb + (int64_t)gi * inner + gr);
                *reinterpret_cast<double2*>(outb + (int64_t)gi * inner + gr) = make_double2(acc[a][b][0], acc[a][b][1]);
            }
        }
    }
}

static long long g_mmt_dmma_launches = 0;
extern "C" long long db_mmt_dmma_launches(void) { return g_mmt_dmma_launches; }

extern "C" int db_mmt_apply(const double* mat, int32_t m, int32_t n, const double* in, double* out, int64_t outer, int64_t inner, void* stream)
{
    if (outer <= 0 || inner <= 0 || m <= 0 || n <= 0) return 0;
    if (outer > 65535) { db_set_error("mmt_apply: outer too large (%lld)", (long long)outer); return 1; }
    const bool aligned = (((uintptr_t)mat | (uintptr_t)in | (uintptr_t)out) & 15) == 0;
    if (aligned && n % 2 == 0 && inner % 2 == 0) {
        dim3 grid((unsigned)((inner + DM_BN - 1) / DM_BN), (unsigned)((m + DM_BM - 1) / DM_BM), (unsigned)outer);
        DB_LAUNCH(k_mmt_dmma, grid, dim3(128), 0, stream, mat, m, n, in, out, inner);
        ++g_mmt_dmma_launches;
        return db_check_launch("mmt_apply(dmma)");
    }
    dim3 grid((unsigned)((inner + MM_BN - 1) / MM_BN), (unsigned)((m + MM_BM - 1) / MM_BM), (unsigned)outer);
    DB_LAUNCH(k_mmt, grid, dim3(256), (MM_BK * MM_BM + MM_BK * MM_BN) * sizeof(double), stream, mat, m, n, in, out, outer, inner);
    return db_check_launch("mmt_apply");
}

// ---------------------------------------------------------------------------------------------------------
// Ragged batch of small dense matrix-vector products (T5): the spin-weighted spherical harmonic colatitude transform
// (reference core/transforms.py:1251-1340) applies a DIFFERENT matrix per azimuthal wavenumber m to the few lines that carry
// that m (cos / -sin pair x tensor components), with the coefficient lines addressed through the folded triangular packing
// (forward or reversed l order).  On the 2-D sphere the work is streaming the matrices (~100 MB per spin weight at Lmax = 254)
// against a handful of right-hand sides, i.e. HBM-bound, not tensor-bound: one warp per output row, lanes along the
// contraction index (coalesced matrix reads), up to RG_C right-hand sides accumulated per pass, shuffle reduction.
//   entry e:  out[o, out_i0 + i, out_row0 + k * out_step, r] = sum_j mat_e[k][j] * in[o, in_i0 + i, in_row0 + j * in_step, r]
//             for k < nrow, j < ncol, i < nm, all o < N0, r < N3;  zero != 0: the output lines are set to zero instead.
// ---------------------------------------------------------------------------------------------------------
#define RG_C 8
#define RG_ROWS 8
__global__ void __launch_bounds__(32 * RG_ROWS)
k_ragged_matvec(const double* __restrict__ mats, const db_ragged_entry* __restrict__ entries, const double* __restrict__ in,
                double* __restrict__ out, int64_t N0, int N1i, int N2i, int N1o, int N2o, int64_t N3)
{
    const db_ragged_entry E = entries[blockIdx.x];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int64_t ncols_total = N0 * E.nm * N3;                  // right-hand sides of this entry
    const double* __restrict__ mat = mats + E.mat_off;
    for (int k = blockIdx.y * RG_ROWS + w; k < E.nrow; k += gridDim.y * RG_ROWS) {
        for (int64_t c0 = 0; c0 < ncols_total; c0 += RG_C) {
            double acc[RG_C];
            int64_t ibase[RG_C], obase[RG_C];
#pragma unroll
            for (int cc = 0; cc < RG_C; ++cc) {
                acc[cc] = 0.0;
                const int64_t c = c0 + cc < ncols_total ? c0 + cc : ncols_total - 1;
                const int64_t r = c % N3; const int64_t t = c / N3; const int i = (int)(t % E.nm); const int64_t o = t / E.nm;
                ibase[cc] = ((o * N1i + E.in_i0 + i) * N2i + E.in_row0) * N3 + r;
                obase[cc] = ((o * N1o + E.out_i0 + i) * N2o + E.out_row0 + (int64_t)k * E.out_step) * N3 + r;
            }
            if (!E.zero) {
                for (int j = lane; j < E.ncol; j += 32) {
                    const double mv = mat[(int64_t)k * E.ncol + j];
                    const int64_t joff = (int64_t)j * E.in_step * N3;
#pragma unroll
                    for (int cc = 0; cc < RG_C; ++cc) acc[cc] = fma(mv, in[ibase[cc] + joff], acc[cc]);
                }
#pragma unroll
                for (int cc = 0; cc < RG_C; ++cc)
#pragma unroll
                    for (int off = 16; off > 0; off >>= 1) acc[cc] += __shfl_down_sync(0xffffffffu, acc[cc], off);
            }
            if (lane == 0) {
#pragma unroll
                for (int cc = 0; cc < RG_C; ++cc)
                    if (c0 + cc < ncols_total) out[obase[cc]] = acc[cc];
            }
        }
    }
}

extern "C" int db_ragged_matvec(const double* mats, const db_ragged_entry* entries, int32_t nentries, int32_t max_nrow,
                                const double* in, double* out, int64_t N0, int32_t N1i, int32_t N2i, int32_t N1o, int32_t N2o, int64_t N3,
                                void* stream)
{
    if (nentries <= 0 || N0 <= 0 || N3 <= 0 || max_nrow <= 0) return 0;
    int yb = (max_nrow + RG_ROWS - 1) / RG_ROWS;
    if (yb > 64) yb = 64;
    DB_LAUNCH(k_ragged_matvec, dim3((unsigned)nentries, (unsigned)yb), dim3(32 * RG_ROWS), 0, stream, mats, entries, in, out, N0, N1i, N2i, N1o, N2o, N3);
    return db_check_launch("ragged_matvec");
}

// ---------------------------------------------------------------------------------------------------------
// Distributed-transpose pack / unpack (X1)
// forward hop (towards grid space): local A (B, n1loc, n2, n3), n2 split in P blocks of n2blk:
//   send[p][b][i][j][r] = A[b][i][p*n2blk + j][r]                       (contiguous per destination rank)
//   after all-to-all rank holds recv[p][b][i][j][r] = rows i of source p -> out (B, n1 = P*n1blk, n2loc, n3):
//   out[b][p*n1blk + i][j][r] = recv[p][b][i][j][r]
// The reverse hop swaps the roles.  Blocks are assumed equal (n2 % P == 0, n1 % P == 0).
// ---------------------------------------------------------------------------------------------------------
// All four permutes move whole contiguous chunks: for fixed (batch b, row i, peer p) the block of `clen` doubles is
// contiguous on both sides.  One CTA (or several, via blockIdx.y) copies one chunk; the only index arithmetic is per chunk.
// Every chunk offset below is a multiple of clen, so with clen even and both base pointers 16-byte aligned every chunk is
// 16-byte aligned on both sides: the host decides that once (vec16) and the chunks are then copied with 128-bit accesses.
//   mode 0 pack    : chunk (b, i, p): src ((b*n1loc + i)*n2 + p*n2blk)*n3        -> dst (((p*B + b)*n1loc + i)*n2blk)*n3,   clen = n2blk*n3
//   mode 1 unpack  : chunk (p, b, i): src (((p*B + b)*n1blk + i)*n2loc)*n3       -> dst ((b*n1 + p*n1blk + i)*n2loc)*n3,    clen = n2loc*n3
//   mode 2 pack_rev: chunk (b, p, i): src ((b*n1 + p*n1blk + i)*n2loc)*n3        -> dst (((p*B + b)*n1blk + i)*n2loc)*n3,   clen = n2loc*n3
//   mode 3 unp_rev : chunk (p, b, i): src (((p*B + b)*n1loc + i)*n2blk)*n3       -> dst ((b*n1loc + i)*n2 + p*n2blk)*n3,    clen = n2blk*n3
struct TrArgs { int64_t B, nA, nB, n3; int P; int mode; int64_t clen; int vec16; };

__global__ void __launch_bounds__(256) k_tr_chunks(const double* __restrict__ src, double* __restrict__ dst, TrArgs a)
{
    const int64_t chunk = blockIdx.x;
    int64_t so, dof;
    if (a.mode == 0) {            // nA = n1loc, nB = n2
        const int64_t p = chunk % a.P; int64_t q = chunk / a.P; const int64_t i = q % a.nA, b = q / a.nA;
        const int64_t n2blk = a.nB / a.P;
        so = ((b * a.nA + i) * a.nB + p * n2blk) * a.n3;
        dof = (((p * a.B + b) * a.nA + i) * n2blk) * a.n3;
    } else if (a.mode == 1) {     // nA = n1, nB = n2loc
        const int64_t n1blk = a.nA / a.P;
        const int64_t i = chunk % n1blk; int64_t q = chunk / n1blk; const int64_t b = q % a.B, p = q / a.B;
        so = (((p * a.B + b) * n1blk + i) * a.nB) * a.n3;
        dof = ((b * a.nA + p * n1blk + i) * a.nB) * a.n3;
    } else if (a.mode == 2) {     // nA = n1, nB = n2loc
        const int64_t n1blk = a.nA / a.P;
        const int64_t i = chunk % n1blk; int64_t q = chunk / n1blk; const int64_t p = q % a.P, b = q / a.P;
        so = ((b * a.nA + p * n1blk + i) * a.nB) * a.n3;
        dof = (((p * a.B + b) * n1blk + i) * a.nB) * a.n3;
    } else {                      // nA = n1loc, nB = n2
        const int64_t n2blk = a.nB / a.P;
        const int64_t i = chunk % a.nA; int64_t q = chunk / a.nA; const int64_t b = q % a.B, p = q / a.B;
        so = (((p * a.B + b) * a.nA + i) * n2blk) * a.n3;
        dof = ((b * a.nA + i) * a.nB + p * n2blk) * a.n3;
    }
    const double* __restrict__ s = src + so;
    double* __restrict__ d = dst + dof;
    const int64_t start = (int64_t)blockIdx.y * blockDim.x + threadIdx.x, stride = (int64_t)gridDim.y * blockDim.x;
    if (a.vec16) {
        DB_CHECK_ALIGN16(s);
        DB_CHECK_ALIGN16(d);
        const double2* __restrict__ s2 = reinterpret_cast<const double2*>(s);
        double2* __restrict__ d2 = reinterpret_cast<double2*>(d);
        for (int64_t e = start; e < (a.clen >> 1); e += stride) d2[e] = s2[e];
    } else {
        for (int64_t e = start; e < a.clen; e += stride) d[e] = s[e];
    }
}

// modes 0 and 3 split nB (= n2) over the P peers, modes 1 and 2 nA (= n1)
static int tr_launch(const double* src, double* dst, int mode, int64_t B, int64_t nA, int64_t nB, int64_t n3, int P, void* stream, const char* name)
{
    if (P < 1) { db_set_error("%s: P must be at least 1 (got %d)", name, P); return 1; }
    const bool split_n2 = mode == 0 || mode == 3;
    if ((split_n2 ? nB : nA) % P) { db_set_error("%s: %s not divisible by P", name, split_n2 ? "n2" : "n1"); return 1; }
    TrArgs a; a.B = B; a.nA = nA; a.nB = nB; a.n3 = n3; a.P = P; a.mode = mode;
    int64_t nchunks;
    if (split_n2) { a.clen = (nB / P) * n3; nchunks = B * nA * P; }
    else { a.clen = nB * n3; nchunks = B * nA; }
    if (nchunks <= 0 || a.clen <= 0) return 0;
    if (nchunks > 2147483647LL) { db_set_error("%s: too many chunks", name); return 1; }
    a.vec16 = (a.clen % 2 == 0) && (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0);
    int64_t gy = (a.clen / 2 + 256 * 8 - 1) / (256 * 8);       // ~8 vector elements per thread
    if (gy < 1) gy = 1;
    if (gy > 64) gy = 64;
    DB_LAUNCH(k_tr_chunks, dim3((unsigned)nchunks, (unsigned)gy), dim3(256), 0, stream, src, dst, a);
    ++g_pw_launches[a.vec16 ? 3 : 4];
    return db_check_launch(name);
}

extern "C" int db_transpose_pack(const double* a, double* sendbuf, int64_t B, int64_t n1loc, int64_t n2, int64_t n3, int32_t P, void* stream)
{
    return tr_launch(a, sendbuf, 0, B, n1loc, n2, n3, P, stream, "transpose_pack");
}
extern "C" int db_transpose_unpack(const double* recvbuf, double* out, int64_t B, int64_t n1, int64_t n2loc, int64_t n3, int32_t P, void* stream)
{
    return tr_launch(recvbuf, out, 1, B, n1, n2loc, n3, P, stream, "transpose_unpack");
}
extern "C" int db_transpose_pack_rev(const double* a, double* sendbuf, int64_t B, int64_t n1, int64_t n2loc, int64_t n3, int32_t P, void* stream)
{
    return tr_launch(a, sendbuf, 2, B, n1, n2loc, n3, P, stream, "transpose_pack_rev");
}
extern "C" int db_transpose_unpack_rev(const double* recvbuf, double* out, int64_t B, int64_t n1loc, int64_t n2, int64_t n3, int32_t P, void* stream)
{
    return tr_launch(recvbuf, out, 3, B, n1loc, n2, n3, P, stream, "transpose_unpack_rev");
}
