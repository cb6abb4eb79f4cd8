/* dedalus_b200 C ABI -- the drop-in boundary for the Dedalus per-timestep hot loop on H100 (sm_90a).
 *
 * Conventions
 *   - every data pointer is a DEVICE pointer (fp64 unless stated; complex = interleaved re,im);
 *     integer "program" arrays are device int32 pointers; `stream` is a cudaStream_t passed as void*;
 *   - return value 0 = success, nonzero = error (message via db_last_error());
 *   - no call synchronises the host; all work is enqueued on `stream`;
 *   - arrays are C-contiguous views (outer, n, inner) with the transform along the middle axis, exactly the
 *     (axis, shape) convention of the reference plugins' forward(gdata, cdata, axis) / backward(...)
 *     (dedalus/core/transforms.py:54-75, basis.py:416-428); input and output buffers must not overlap.
 *
 * Each entry point cites the reference interface it replaces (paths relative to the reference repo).
 */
#ifndef DEDALUS_B200_H
#define DEDALUS_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

const char* db_last_error(void);
int db_version(void);
/* device / arch probe: returns compute capability major*10+minor of the current device, <0 on error */
int db_device_arch(void);

/* ---------------------------------------------------------------------------------------------------------
 * Spectral transforms (T1-T4).  A "plan" is a small table block built by the host (dedalus_b200/fftplan.py)
 * and uploaded once: radices, twiddles, digit-reversal permutation.
 * ------------------------------------------------------------------------------------------------------- */
typedef struct {
    int32_t n;            /* transform length on the grid (real length for real transforms)          */
    int32_t nc;           /* length of the in-shared-memory complex FFT (n/2 for even real, n else)   */
    int32_t half;         /* 1 if the real transform uses the half-length complex trick (n even)      */
    int32_t nrad;         /* number of radix passes                                                   */
    int32_t rad[16];      /* radices, DIF order                                                       */
    const double* tw;     /* [nc][2]  exp(-2 pi i j / nc)                                             */
    const double* twr;    /* [nc+1][2] exp(-2 pi i k / n)   (real <-> half-complex post/pre twiddle)   */
    const double* twq;    /* [n][2]  exp(-i pi k / (2n))    (DCT quarter-wave twiddle)                 */
    const int32_t* perm;  /* [nc] frequency index held at position p after the DIF passes            */
    const int32_t* iperm; /* [nc] position holding frequency k (inverse of perm)                      */
    const double* twn;    /* [n][2]  exp(-2 pi i j / n)     (register-resident two-stage kernels)      */
} db_fft_plan;

/* Real Fourier, cos/-sin interleaved coefficients, unit-amplitude normalisation, Nyquist dropped.
 * Replaces FFTWRealFFT.forward/backward + RealFFT.unpack_rescale/repack_rescale
 * (core/transforms.py:469-509, 537-565; libraries/fftw/fftw_wrappers.pyx:141-154, 188-207).
 * g: (outer, n_grid, inner) real;  c: (outer, n_coeff, inner) real.
 * backward: `deriv` >= 0 applies (d/dx)^deriv in coefficient space first, wavenumber spacing `kscale`
 * (fuses DifferentiateRealFourier, core/basis.py:1203-1224, into the transform's load stage). */
/* diagnostic: number of db_rfft_* calls served by the register-resident kernels (csrc/rfft_regs.cu) so far */
long long db_rfft_regs_launches(void);
int db_rfft_forward(const db_fft_plan* plan, const double* g, double* c, int64_t outer, int32_t n_coeff, int64_t inner, void* stream);
int db_rfft_backward(const db_fft_plan* plan, const double* c, double* g, int64_t outer, int32_t n_coeff, int64_t inner,
                     int32_t deriv, double kscale, void* stream);

/* The same transforms with BLOCKED row addressing on either side, so that the pencil transposes (X1) need no pack /
 * unpack kernels: with rpb > 0 row r of outer index o lives at (r / rpb) * blk_stride + (o * rpb + r % rpb) * inner
 * (elements) -- the rows are grouped into the per-peer blocks of an all-to-all buffer: the transform before the exchange
 * writes the send buffer directly (out_rpb = rows per peer), the transform after it reads the receive buffer directly
 * (in_rpb).  Replaces the copies in and out of the transpose buffers of FFTWTranspose (core/transposes.pyx:146-246).
 * rpb = 0: plain layout on that side.  Returns 2 (no error recorded) when the size / layout is not covered by the
 * register-resident kernels (dealiased sizes, inner % 16 == 0): the caller then uses db_transpose_* + the plain entries. */
int db_rfft_forward_blocked(const db_fft_plan* plan, const double* g, double* c, int64_t outer, int32_t n_coeff, int64_t inner,
                            int32_t in_rpb, int64_t in_blk_stride, int32_t out_rpb, int64_t out_blk_stride, void* stream);
int db_rfft_backward_blocked(const db_fft_plan* plan, const double* c, double* g, int64_t outer, int32_t n_coeff, int64_t inner,
                             int32_t deriv, double kscale,
                             int32_t in_rpb, int64_t in_blk_stride, int32_t out_rpb, int64_t out_blk_stride, void* stream);

/* The all-to-all of a pencil transpose as the transform's OWN stores into peer memory (X1 without a library collective;
 * replaces fftw_mpi_execute_r2r on the transposed plan, core/transposes.pyx:173-192, 209, 223): as the _blocked entries, but
 * output block b (the rows destined for GPU b) is written to out_blocks[b] -- GPU b's receive buffer mapped into this process
 * (NVLink peer memory, e.g. the buffer_ptrs of a torch symmetric-memory allocation) -- instead of the local send buffer, so
 * the exchange overlaps the arithmetic tile by tile and no communication kernel is launched.  out_blocks is a HOST array of
 * n_peers (<= 8) device pointers (copied into the launch); local_out is only the 16-byte aligned origin of the column offsets.
 * The caller orders the consumers after all writers with a device-side barrier (signal pads).  Returns 2 if not covered. */
int db_rfft_forward_peer(const db_fft_plan* plan, const double* g, double* local_out, int64_t outer, int32_t n_coeff, int64_t inner,
                         int32_t in_rpb, int64_t in_blk_stride, int32_t out_rpb, int32_t n_peers, double* const* out_blocks, void* stream);
int db_rfft_backward_peer(const db_fft_plan* plan, const double* c, double* local_out, int64_t outer, int32_t n_coeff, int64_t inner,
                          int32_t deriv, double kscale, int32_t in_rpb, int64_t in_blk_stride, int32_t out_rpb,
                          int32_t n_peers, double* const* out_blocks, void* stream);

/* Complex Fourier, ordering [0..KM,(Nyq),-KM..-1], forward scaled by 1/N.
 * Replaces FFTWComplexFFT (core/transforms.py:243-267, 302-330).  Arrays are interleaved complex. */
int db_cfft_forward(const db_fft_plan* plan, const double* g, double* c, int64_t outer, int32_t n_coeff, int64_t inner, void* stream);
int db_cfft_backward(const db_fft_plan* plan, const double* c, double* g, int64_t outer, int32_t n_coeff, int64_t inner,
                     int32_t deriv, double kscale, void* stream);

/* Chebyshev / ultraspherical transforms on the Gauss-Chebyshev grid: DCT-II / DCT-III with the Jacobi
 * unit-weight normalisation, sign flip of odd modes, truncation / zero padding, and optional banded
 * spectral matrices.  Replaces FFTWFastChebyshevTransform (core/transforms.py:715-746, 771-902) and the
 * apply_sparse / solve_upper_sparse calls inside it (tools/linalg.pyx:20-82, 189-258).
 * Banded matrices are upper triangular, stored by diagonals: diag[d][i] = A[i][i+d], d < ndiag, row length n_coeff.
 *   forward : coefficients = conv_apply( truncate( scale( DCT-II(g) ) ) )        (conv_ndiag = 0: none)
 *   backward: g = DCT-III( scale( solve_upper(conv_solve, apply(pre_apply, c)) ) ) (either may be absent);
 *             row 0 of solve_diags holds the RECIPROCAL of the diagonal. */
int db_cheb_forward(const db_fft_plan* plan, const double* g, double* c, int64_t outer, int32_t n_coeff, int64_t inner,
                    const double* conv_diags, int32_t conv_ndiag, void* stream);
int db_cheb_backward(const db_fft_plan* plan, const double* c, double* g, int64_t outer, int32_t n_coeff, int64_t inner,
                     const double* pre_diags, int32_t pre_ndiag, const double* solve_diags, int32_t solve_ndiag, void* stream);

/* db_cheb_backward on contiguous lines with the derivative pre-apply (pre_ndiag <= 3) and the back-substitution of a
 * conversion that has only its main and second super-diagonal fused in (solve2_diags: [2][n_coeff], row 0 = reciprocal
 * diagonal, row 1 = second super-diagonal -- the stride-2 storage of db_band_lines).  Same result as db_band_lines followed
 * by db_cheb_backward, without the intermediate array.  Returns 2 (and records no error) when the size / alignment is
 * not covered by the fused kernel. */
int db_cheb_backward_scan(const db_fft_plan* plan, const double* c, double* g, int64_t lines, int32_t n_coeff,
                          const double* pre_diags, int32_t pre_ndiag, const double* solve2_diags, void* stream);

/* Banded coefficient-space work along CONTIGUOUS lines (inner == 1), used ahead of db_cheb_backward when a spectral
 * derivative / ultraspherical back-conversion is fused in: out = solve_upper(solve_diags, apply(pre_diags, in)).
 * One thread per line with the line staged in shared memory: decouples the O(n) serial recurrence from the FFT
 * kernel's CTA shape (core/transforms.py:876-884 solve_upper_sparse; tools/linalg.pyx:20-82).
 * Diagonal storage as in db_cheb_backward (row 0 of solve_diags = reciprocal diagonal). */
int db_band_lines(const double* in, double* out, int64_t lines, int32_t n,
                  const double* pre_diags, int32_t pre_ndiag, const double* solve_diags, int32_t solve_ndiag,
                  int32_t solve_stride, void* stream);

/* Dense matrix transform along an axis: out(o, i, r) = sum_j mat[i][j] * in(o, j, r).
 * Replaces SeparableMatrixTransform -> apply_dense (core/transforms.py:54-75, tools/array.py:104-129). */
int db_mmt_apply(const double* mat, int32_t m, int32_t n, const double* in, double* out, int64_t outer, int64_t inner, void* stream);
/* diagnostic: number of db_mmt_apply calls served by the FP64 tensor-core kernel so far (n and inner even, mat / in / out 16-byte
 * aligned); every other call runs the FMA-pipe kernel */
long long db_mmt_dmma_launches(void);

/* Ragged batch of dense matrix-vector products: the spin-weighted spherical harmonic colatitude transform.
 * Replaces SWSHColatitudeTransform.forward_reduced / backward_reduced (core/transforms.py:1263-1290): for every local
 * azimuthal wavenumber m (one entry; m_maps of core/basis.py:2940-2970) the matrix of that m (`mats + mat_off`, row-major
 * nrow x ncol; built by the host as core/transforms.py:1296-1340) is applied along axis 2 of the reduced 4-D views
 *   in (N0, N1i, N2i, N3),  out (N0, N1o, N2o, N3)
 * to the nm lines in_i0 .. in_i0 + nm of axis 1 (cos / -sin pair), reading input row in_row0 + j * in_step and writing
 * output row out_row0 + k * out_step (steps of -1 address the folded, reversed-l halves of the triangular packing);
 * zero != 0: the nm output lines (rows out_row0 + k * out_step, k < nrow) are set to zero (|m| > Lmax on the way back). */
typedef struct {
    int64_t mat_off;
    int32_t nrow, ncol;
    int32_t in_i0, in_row0, in_step;
    int32_t out_i0, out_row0, out_step;
    int32_t nm, zero;
} db_ragged_entry;
int db_ragged_matvec(const double* mats, const db_ragged_entry* entries, int32_t nentries, int32_t max_nrow,
                     const double* in, double* out, int64_t N0, int32_t N1i, int32_t N2i, int32_t N1o, int32_t N2o, int64_t N3,
                     void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Grid-space products (P1): every output is a sum of coef * product of inputs, evaluated pointwise.
 * Replaces DotProduct.operate / MultiplyFields.operate / AddFields.operate chains
 * (core/arithmetic.py:246-251, 666-674, 855-866).
 * in: (n_in, npoints) stacked inputs, out: (n_out, npoints).  Program: for output o, terms
 * term_ptr[o]..term_ptr[o+1]; term t has coefficient coef[t] and factors fac[fac_ptr[t]..fac_ptr[t+1]).
 * At most 113 inputs (a tile of 256 points of every input in shared memory); more return 1 with a message.  An even npoints with
 * 16-byte aligned in and out and at most 56 inputs takes the double-buffered two-points-per-thread kernel, everything else the
 * single-buffered one; both evaluate the same arithmetic, so their results are bitwise equal.  npoints <= 0 or n_out <= 0: nothing. */
int db_pointwise(const double* in, double* out, int64_t npoints, int32_t n_in, int32_t n_out,
                 const int32_t* term_ptr, const double* coef, const int32_t* fac_ptr, const int32_t* fac, int32_t nfac_total,
                 void* stream);
/* The same for programs whose terms have one or two factors (quadratic nonlinearities): term t of output o
 * (term_ptr[o] <= t < term_ptr[o+1]) is coef * in[a] * in[b], or coef * in[a] when b < 0, accumulated as fma(coef * in[a], in[b], acc).
 * npoints even, at most 56 inputs, and in, out and terms 16-byte aligned (terms are read as 16-byte records); otherwise returns 1
 * with a message. */
typedef struct { double coef; int32_t a; int32_t b; } db_pair_term;
int db_pointwise_pairs(const double* in, double* out, int64_t npoints, int32_t n_in, int32_t n_out,
                       const int32_t* term_ptr, const db_pair_term* terms, void* stream);
/* The x pass of a quadratic right-hand side fused with its products (real Fourier x axis, n in 24, 48, 96, 192, 384):
 * backward x transforms of the inputs, the products, and the forward x transforms of the outputs, one tile of 16 lines at a time,
 * with no grid array in global memory.  in: stack of (n_coeff, inner) coefficient arrays, input s at in + s * in_stride;
 * out: output o at out + o * out_stride, (n_coeff, inner).  The schedule (device arrays) is walked once per tile:
 *   item with DB_XPROD_HELD: transform input `src` with x derivative `deriv` and keep its grid values as held factor `a` (0..2);
 *   other items: one term coef * a * b (b < 0: coef * a) of output `out`, factors coded 0..2 = held, 3 = input `src` transformed
 *   just before (src < 0: no transform), accumulated exactly as db_pointwise_pairs does; DB_XPROD_LAST after an output's last term.
 * loads: the src of every item with src >= 0, in item order.  inner % 16 == 0, arrays 16-byte aligned, n_held <= 3. */
typedef struct { double coef; int32_t src; int32_t deriv; int32_t a; int32_t b; int32_t out; int32_t flags; } db_xprod_item;
#define DB_XPROD_HELD 1
#define DB_XPROD_LAST 2
int db_rfft_x_products(const db_fft_plan* plan, const double* in, int64_t in_stride, double* out, int64_t out_stride,
                       int32_t n_coeff, int64_t inner, double kscale, const db_xprod_item* items, int32_t n_items,
                       const int32_t* loads, int32_t n_loads, int32_t n_held, void* stream);
/* CTAs resident per SM (cudaOccupancyMaxActiveBlocksPerMultiprocessor on the current device) of the register real-Fourier
 * transforms at n grid points: kind 0 backward, 1 forward, 2 the fused x pass with n_coeff rows and n_held held factors (its
 * persistent grid is this many CTAs per SM).  -1 where there is no such kernel. */
int db_rfft_blocks_per_sm(int32_t kind, int32_t n, int32_t n_coeff, int32_t n_held);

/* ---------------------------------------------------------------------------------------------------------
 * Pencil systems (S1-S4).  A batch holds S structurally identical systems of size n; one thread owns one system.
 * Every [rows][systems] array (vectors: rows = n; factors: rows = n_entries) is stored TILE-MAJOR:
 *     element (i, s)  at  ((s / DB_TILE) * rows + i) * DB_TILE + (s % DB_TILE),      DB_TILE = 64
 * so each group of 64 systems owns one contiguous slab (coalesced across systems, sequential along rows / entries).
 * Arrays are allocated for ceil(S / DB_TILE) tiles.  `ld` (>= S) is the stride of the small per-system tables
 * (mono_vals[m*ld + s], sys_off[kind*ld + s]).
 * ------------------------------------------------------------------------------------------------------- */
/* gather: field arena -> pencil vectors (Subproblem.gather_inputs/gather_outputs, core/subsystems.py:340-362)
 * scatter: pencil vectors -> field arena (Subproblem.scatter_inputs, core/subsystems.py:364-371).
 * Line q: arena offset line_base[q] + sys_off[line_kind[q]*ld_sys + s] + m  <->  vec element (line_pos[line_ptr[q]+m], s). */
int db_pencil_gather(const double* arena, double* vec, int32_t S, int32_t n, int32_t nlines, int32_t max_len,
                     const int64_t* line_base, const int32_t* line_kind, const int32_t* line_ptr, const int32_t* line_pos,
                     const int64_t* sys_off, int32_t ld_sys, void* stream);
int db_pencil_scatter(const double* vec, double* arena, int32_t S, int32_t n, int32_t nlines, int32_t max_len,
                      const int64_t* line_base, const int32_t* line_kind, const int32_t* line_ptr, const int32_t* line_pos,
                      const int64_t* sys_off, int32_t ld_sys, void* stream);

/* y = A(k) x with A(k) = sum_mono mono_vals[mono][s] * T_mono, CSR-by-row term lists
 * (apply_sparse(sp.M_min / sp.L_min, X): core/timesteppers.py:144-147, 590-591, 604; tools/linalg.pyx:284-303).
 * Either output may be NULL. */
int db_pencil_matvec(int32_t n, int32_t S, int32_t ld, const double* mono_vals, const double* x,
                     const int32_t* m_ptr, const int32_t* m_col, const int32_t* m_mono, const double* m_val, double* y_m,
                     const int32_t* l_ptr, const int32_t* l_col, const int32_t* l_mono, const double* l_val, double* y_l,
                     void* stream);

/* LHS assembly from templates, LU = a0*M + b0*L on the static fill pattern
 * (sp.LHS = a0*sp.M_min + b0*sp.L_min: core/timesteppers.py:173-180, 632-639). */
int db_pencil_assemble(double* lu, int32_t n_entries, int32_t S, int32_t ld, const double* mono_vals,
                       const int32_t* asm_ptr, const int32_t* asm_mono, const double* asm_val, void* stream);

/* in-place LU without pivoting on the static ordering (matsolver construction: libraries/matsolvers.py:126-157).
 * info[0] receives the number of systems that hit a zero / non-finite pivot. */
int db_pencil_factor(double* lu, int32_t n, int32_t S, int32_t n_entries, const int32_t* diag_eid,
                     const int32_t* fl_ptr, const int32_t* fl_eid, const int32_t* fu_ptr, const int32_t* fu_eid,
                     const int32_t* fd_eid, int32_t* info, void* stream);

/* x = LU^{-1} ( sum_j coef[j] * vecs[j] ): the right-hand-side combination of the IMEX schemes is fused into
 * the load (RHS build core/timesteppers.py:156-166, 617-623; solve 182-184, 641-642; matsolvers.py:141-157). */
#define DB_TILE 64

typedef struct {
    int32_t nvec;
    const double* vec[16];
    double coef[16];
} db_lincomb;
int db_pencil_solve(const double* lu, int32_t n, int32_t S, int32_t ld,
                    const int32_t* prog, int32_t n_fwd, int32_t n_entries,
                    const db_lincomb* rhs, double* x, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Fused launches over ALL batches of a solver ("batch set").  The per-stage pencil work of one IMEX stage is then
 * 4 launches (mat-vec, gather F, solve, scatter) however many classes / parity components the problem has, and small
 * batches (kx = 0 or ky = 0 pencils) run concurrently with the large ones instead of serialising on the stream.
 * `batches` is a DEVICE array of db_batch built once by the host; per-call arguments are slot indices.
 * The solve program is a flat instruction stream aligned one-to-one with the LU value stream: a forward section
 * then a backward section, each padded to a multiple of 16 entries.  First x <- right-hand-side combination; then
 *   c >= 0            : acc -= LU[e] * x[c]            (c = column * DB_TILE, element offset of that row in a vector)
 *   c < 0, != DB_I_SKIP: leave the current row (forward: x[row] = acc; backward: x[row] = acc * LU[e], the reciprocal
 *                       pivot) and enter row (-1 - c) / DB_TILE with acc = x[row].  The first entry of a section only
 *                       enters a row.  A forward row may be left and re-entered (its partial sum lives in x[row]).
 *   DB_I_SKIP         : padding (factor value 0)
 * Rows are visited in LEVEL order of the triangular solve's dependency DAG (rows of one level are independent); runs
 * of dense forward rows (boundary rows) are interleaved in 15-entry segments so the run sweeps x once, not once per row.
 * The fused kernel consumes the stream through per-chunk control blocks (`ctrl`, built by the host from the stream).
 * ------------------------------------------------------------------------------------------------------- */
#define DB_MAX_VECS 24
#define DB_MAX_LU 4
#define DB_I_SKIP ((int32_t)0x80000000)
/* one term of a template mat-vec: y[row] += val * mono[mono][s] * x[column][s]; in the fused kernel's record arrays col_off is
 * the row inside the block's shared-memory window or column * DB_TILE (see db_batch.m_split) */
typedef struct { double val; int32_t col_off; int32_t mono; } db_term;
typedef struct {
    int32_t n, S, ld, n_entries;       /* S pencils; every pencil carries `nrhs` systems sharing ONE factorisation (see nrhs) */
    int32_t n_fwd, n_bwd;
    int32_t blk_solve, blk_matvec, blk_move[2], blk_assemble;   /* first block of this batch in each fused launch */
    int32_t nlines[2], max_len[2];
    const int32_t* prog;
    const double* mono;
    double* vec[DB_MAX_VECS];
    double* lu[DB_MAX_LU];
    const int32_t *m_ptr, *m_col, *m_mono; const double* m_val;
    const int32_t *l_ptr, *l_col, *l_mono; const double* l_val;
    const db_term *m_rec, *l_rec;      /* the same term lists packed 16 bytes per term (fused mat-vec kernel) */
    const int32_t* ctrl;               /* [n_entries/16][36] per-chunk control blocks of the branch-free solve kernel:
                                          gather offsets[16], finished-row offsets[16], masks end / begin / late / late for a one-chunk-early gather */
    int32_t n_mono;
    int32_t mv_rows;                   /* rows per CTA of the fused mat-vec (= 32, MV_R in csrc/pencil.cu) */
    const int32_t* mv_win;             /* [ceil(n / mv_rows)][2]: first x row and row count (<= 80) of the shared-memory window of each row block */
    const int32_t *m_split, *l_split;  /* [n]: within row i, records m_ptr[i]..split[i] lie inside the window (col_off = window row),
                                          records split[i]..m_ptr[i+1] outside (col_off = column * DB_TILE)                       */
    const int64_t* line_base[2]; const int32_t* line_kind[2]; const int32_t* line_ptr[2]; const int32_t* line_pos[2];
    const int64_t* sys_off[2];
    /* Merged sign-equivalent components.  The real-Fourier parity blocks of a pencil (cos/cos, cos/sin, ... : the reference
     * keeps them inside one SuperLU system per pencil, core/subsystems.py:497-602) have matrices A_c = D1_c A_0 D2_c with
     * D = diag(+-1); stored as D2_c x_c / D1_c b_c they are `nrhs` right-hand sides of the SAME matrix A_0.  Work vectors
     * then hold nrhs * ld columns, member c of pencil s in column c * ld + s (tile-major over that column index); the
     * factors hold ld columns.  line_base and line_sign are [nrhs][nlines]: arena offset and sign of member c's line q. */
    int32_t nrhs;
    const double* line_sign[2];
    /* factorisation programs */
    const int32_t *diag_eid, *fl_ptr, *fl_eid, *fu_ptr, *fu_eid, *fd_eid;
    const int32_t *asm_ptr, *asm_mono; const double* asm_val;
    int32_t* info;
} db_batch;

typedef struct {
    int32_t nvec;
    int32_t slot[16];
    double coef[16];
} db_slotcomb;

/* side: 0 = variables/state arena (columns), 1 = equations arena (rows); gather != 0: arena -> vec[slot], else vec[slot] -> arena */
int db_batches_move(const db_batch* batches, int32_t nbatch, int32_t total_blocks, int32_t side, int32_t gather,
                    int32_t slot, double* arena, void* stream);
/* vec[ym_slot] = M vec[x_slot], vec[yl_slot] = L vec[x_slot]; a negative slot skips that product */
int db_batches_matvec(const db_batch* batches, int32_t nbatch, int32_t total_blocks, int32_t x_slot, int32_t ym_slot, int32_t yl_slot, void* stream);
/* vec[x_slot] = LU[lu_slot]^{-1} (sum_j coef[j] vec[slot[j]]), 1 <= nvec <= 16 */
/* max_nrhs: largest db_batch.nrhs of the set (the CTAs have 64 * max_nrhs threads) */
int db_batches_solve(const db_batch* batches, int32_t nbatch, int32_t total_blocks, int32_t max_nrhs, int32_t lu_slot, int32_t x_slot,
                     const db_slotcomb* rhs, void* stream);
/* Kernel and ring of db_batches_solve for this process (also environment DB_SOLVE_WS / _PIPE / _RT / _DEEP / _STAGES / _CPS /
 * _MINB / _PF / _DEEP_MPC, read once).  kernel: 0 warp-specialised ring (default), 1 flat, 2 pipelined gathers, 3 / 4 two / four
 * members per thread (these solve whole groups of 2 / 4 members: the work vectors must hold them), 5 deep prefetch.  stages: ring
 * depth, 2 .. 24 (deep: at least 5); chunks_per_stage: 1 .. 8 (warp-specialised ring only); minb: 1 .. 4, the CTAs per SM the
 * register budget is built for; prefetch: 0 none, 1 L2, 2 L1 prefetch of row start values; deep_members: 1, 2 or 4 members per
 * CTA of the deep kernel.  All variants give bitwise-equal results.  A negative field returns to the environment's choice.
 * Out-of-range values, and rings that do not fit in shared memory, are rejected (here or by the next solve) with an error. */
int db_batches_solve_set_mode(int32_t kernel, int32_t stages, int32_t chunks_per_stage, int32_t minb, int32_t prefetch, int32_t deep_members);
/* LU[lu_slot] = assembled LHS (asm_* programs), then in-place factorisation */
int db_batches_assemble(const db_batch* batches, int32_t nbatch, int32_t total_blocks, int32_t lu_slot, void* stream);
int db_batches_factor(const db_batch* batches, int32_t nbatch, int32_t total_blocks, int32_t lu_slot, void* stream);

/* Verification of a factorisation with a probe right-hand side: given b = vec[b_slot], x = LU^{-1} b (db_batches_solve) and
 * vec[m_slot] = M x, vec[l_slot] = L x (db_batches_matvec), writes per system (index = solve block * 64 + lane, padding lanes 0)
 *     max_i |a0 (Mx)_i + b0 (Lx)_i - b_i| / (max|b| + max|a0 Mx| + max|b0 Lx|)       (+inf if anything is non-finite)
 * No reference counterpart: the reference's SuperLU pivots each pencil on its own (libraries/matsolvers.py:126-183); a pivot
 * order shared by a whole batch must be checked for every member after each factorisation (core/timesteppers.py:632-639). */
int db_batches_residual(const db_batch* batches, int32_t nbatch, int32_t total_blocks, int32_t b_slot, int32_t m_slot,
                        int32_t l_slot, double a0, double b0, double* out, void* stream);

/* out = sum_j coef[j]*vecs[j] over `count` doubles (explicit RHS build, used by tests and diagnostics). */
int db_lincomb_apply(const db_lincomb* terms, double* out, int64_t count, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Distributed transpose pack / unpack (X1): local permutes either side of the NCCL all-to-all.
 * Replaces the np.copyto pack/unpack around fftw_mpi_plan_many_transpose (core/transposes.pyx:106-113, 211-246).
 * A: (B, N1loc, N2, N3) -> send buffer (P, B, N1loc, N2blk, N3); recv (P, B, N1blk, N2loc, N3) -> (B, N1, N2loc, N3). */
int db_transpose_pack(const double* a, double* sendbuf, int64_t B, int64_t n1loc, int64_t n2, int64_t n3, int32_t P, void* stream);
int db_transpose_unpack(const double* recvbuf, double* out, int64_t B, int64_t n1, int64_t n2loc, int64_t n3, int32_t P, void* stream);
int db_transpose_pack_rev(const double* a, double* sendbuf, int64_t B, int64_t n1, int64_t n2loc, int64_t n3, int32_t P, void* stream);
int db_transpose_unpack_rev(const double* recvbuf, double* out, int64_t B, int64_t n1loc, int64_t n2, int64_t n3, int32_t P, void* stream);
/* All four: P >= 1 and the split axis (n2 for pack / unpack_rev, n1 for unpack / pack_rev) divisible by P, else 1 with a message;
 * B, n1 or n3 = 0: nothing.  A chunk (n2blk * n3 or n2loc * n3 doubles) is copied with 16-byte accesses when its length is even and
 * both base pointers are 16-byte aligned, with 8-byte accesses otherwise. */

/* diagnostic: launches so far of the kernels behind db_pointwise, db_pointwise_pairs and the transposes, by kind: 0 the
 * single-buffered general kernel, 1 the double-buffered general kernel, 2 the pairs kernel, 3 a transpose with 16-byte accesses,
 * 4 a transpose with 8-byte accesses; -1 for any other kind */
long long db_pointwise_launches(int32_t kind);

/* ---------------------------------------------------------------------------------------------------------
 * Curvilinear pencil path (SURVEY section 8f rank 2: sphere / shell problems).  On the sphere the pencils are one system
 * per azimuthal wavenumber m, coupled along the degree l (core/basis.py:2780-2786 matrix_dependence; operators
 * core/basis.py:3299-3420, core/operators.py:2995-3050 MulCosine, 2125-2160 SpinSkew): RAGGED sizes, narrow bands.
 * They are stored in LAPACK's general-band layout, column-major,
 *     operator storage (ld0 = kl + ku + 1):    A(i, j) at ab0[op_off + (ku + i - j) + j * ld0]
 *     factor storage   (ldf = 2 kl + ku + 1):  A(i, j) at ab [lu_off + (kl + ku + i - j) + j * ldf]
 * and factorised with row interchanges by one warp per system (replaces the per-pencil SuperLU of
 * libraries/matsolvers.py:126-183 driven from core/timesteppers.py:577-583, 632-639).  Vectors of system s hold nrhs
 * right-hand-side columns: element (i, r) at vec_off + i * nrhs + r.
 * ------------------------------------------------------------------------------------------------------- */
typedef struct {
    int32_t n, nrhs;
    int64_t op_off;       /* offset (doubles) of this system's band in the operator-storage buffers (M, L)      */
    int64_t lu_off;       /* offset (doubles) in the factor-storage buffer                                        */
    int64_t piv_off;      /* offset (int32) of its pivot rows                                                      */
    int64_t vec_off;      /* offset (doubles) of its rows in every work vector                                     */
} db_banded_sys;
typedef struct { int32_t nvec; const double* vec[16]; double coef[16]; } db_veccomb;
/* lu = a0 * M + b0 * L (fill-in rows zeroed): the LHS of an IMEX stage, core/timesteppers.py:632-639 */
int db_banded_combine(const db_banded_sys* sys, int32_t nsys, int32_t kl, int32_t ku, double a0, const double* m_ab,
                      double b0, const double* l_ab, double* lu, void* stream);
/* in-place band LU with partial pivoting of every system; info[s] = zero / non-finite pivots met */
int db_banded_factor(const db_banded_sys* sys, int32_t nsys, int32_t kl, int32_t ku, double* lu, int32_t* ipiv, int32_t* info, void* stream);
/* x = A^{-1} (sum_k coef_k vec_k) for all columns (the RHS combination of core/timesteppers.py:617-623 fused in);
 * x may be one of the vec_k.  max_n / max_nrhs: largest n / nrhs over the systems. */
int db_banded_solve(const db_banded_sys* sys, int32_t nsys, int32_t kl, int32_t ku, int32_t max_n, int32_t max_nrhs,
                    const double* lu, const int32_t* ipiv, const db_veccomb* rhs, double* x, void* stream);
/* ya = A x and / or yb = B x (operator storage; either output may be NULL): M.X, L.X of core/timesteppers.py:590-591 */
int db_banded_matvec(const db_banded_sys* sys, int32_t nsys, int32_t kl, int32_t ku, const double* a_ab, const double* b_ab,
                     const double* x, double* ya, double* yb, void* stream);
/* gather (vec[e] = idx[e] >= 0 ? arena[idx[e]] : 0) / scatter (arena[idx[e]] = vec[e] where idx[e] >= 0) through an index
 * table: pencil vectors <-> coefficient arrays in the folded triangular (m, l) packing (core/subsystems.py:340-371) */
int db_index_move(const int64_t* idx, int64_t count, double* arena, double* vec, int32_t gather, void* stream);

/* the same for runs of `run` contiguous doubles per index entry (row permutations around the curvilinear transposes) */
int db_index_move_runs(const int64_t* idx, int64_t count, int64_t run, double* arena, double* vec, int32_t gather, void* stream);

/* Dense batches with many right-hand sides: the per-degree pencil systems of spherical-shell problems -- ONE matrix per l for all
 * m <= l (core/subsystems.py:272-274: Subproblem.shape = (n, n_subsystems); libraries/matsolvers.py:126-183 per matrix).  Matrices
 * [nsys][n][n] row-major, every system padded to the same n; vectors of system s: element (i, r) at vec_off + i * ncols + r. */
typedef struct { int32_t ncols; int32_t pad; int64_t vec_off; } db_dense_sys;
int db_dense_combine(int32_t nsys, int32_t n, double a0, const double* m, double b0, const double* l, double* out, void* stream);
/* in-place LU with partial pivoting, one CTA per system; ipiv [nsys][n], info[s] = zero / non-finite pivots met */
int db_dense_factor(int32_t nsys, int32_t n, double* a, int32_t* ipiv, int32_t* info, void* stream);
/* x = A^{-1} (sum_k coef_k vec_k) for every column of every system (x must not be one of the vec_k) */
int db_dense_solve(const db_dense_sys* sys, int32_t nsys, int32_t n, int32_t max_ncols, const double* lu, const int32_t* ipiv,
                   const db_veccomb* rhs, double* x, void* stream);
/* ya = A x and / or yb = B x (either output may be NULL) */
int db_dense_matvec(const db_dense_sys* sys, int32_t nsys, int32_t n, const double* a, const double* b, const double* x,
                    double* ya, double* yb, void* stream);

/* the same products with the operators in CSR (ptr [nsys][n + 1], offsets into col / val global over the batch): the pencil
 * operators M, L of shell problems are a few percent dense, only their factors fill in */
int db_csr_matvec(const db_dense_sys* sys, int32_t nsys, int32_t n, const int64_t* a_ptr, const int32_t* a_col, const double* a_val,
                  const int64_t* b_ptr, const int32_t* b_col, const double* b_val, const double* x, double* ya, double* yb, void* stream);

/* Complex linear combinations on (cos, -sin) pairs.  in / out: (ncomp, 2 * npair, ncol), rows 2j and 2j + 1 = real and
 * imaginary part of the exp(i m phi) coefficient (core/basis.py:1108-1134).  Output o = sum over its terms
 * term_ptr[o] <= t < term_ptr[o + 1] of (re + i im) * sym * in[src], sym = syms[sym_off + (j * ncol + c) / sym_div] or 1 (sym_off < 0);
 * sym_div > 1 when the symbol is constant along the trailing sym_div entries of a row (the radial index of shell data: the
 * regularity recombination Q(l) of core/basis.py:3590-3627).
 * Replaces (a) SeparableSphereOperator.operate -- SphereGradient / Divergence / Laplacian symbols k(l, s, mu) / R
 * (core/operators.py:2725-2866, core/basis.py:3299-3420) and SpinSkew (core/operators.py:2125-2160) in coefficient space,
 * (b) the component <-> spin recombination (libraries/spin_recombination.pyx:9-56 with U of core/coords.py:219-232) in
 * (azimuthal coefficient, colatitude grid) space.  in and out must not overlap. */
typedef struct { double re, im; int64_t sym_off; int32_t src; int32_t pad; } db_pair_lin_term;
int db_pair_lincomb(const double* in, double* out, int64_t npair, int64_t ncol, int32_t n_out,
                    const int32_t* term_ptr, const db_pair_lin_term* terms, const double* syms, int64_t sym_div, void* stream);

/* max |x| reduction (CFL / flow properties; extras/flow_tools.py:33-37 before the Allreduce).
 * The three reductions below ACCUMULATE: out = max(out, maximum over the input), so `out` is zero-initialised before the first call
 * and may be passed on from one field to the next; a value already larger stays.  A NaN anywhere in the input (or already in
 * `out`) gives NaN, as np.max does, and an infinite value gives +inf: a field that has blown up never yields a finite maximum. */
int db_absmax(const double* x, int64_t count, double* out, void* stream);

/* Advective CFL frequency: out = max over grid points of sum_i |u_i| * inv_dx_i[index along axis i]
 * (operators.AdvectiveCFL, core/operators.py:4342-4400, basis.py:6078-6112, followed by the max of
 * extras/flow_tools.py:191-214).  u_i: ncomp grid arrays of shape (g0, g1, g2) (use 1 for missing axes);
 * inv_dx_i: device vectors of the local inverse grid spacings along axis i.  `out` must be zero-initialised. */
int db_cfl_max(const double* const* u, const double* const* inv_dx, int32_t ncomp, int64_t g0, int64_t g1, int64_t g2,
               double* out, void* stream);

/* The same on spheres / spherical shells: max of sqrt(u_phi^2 + u_theta^2) * inv_h[ir] + |u_r| * inv_dr[ir] over arrays of shape
 * (n_ang, n_r); inv_h = sqrt(Lmax (Lmax + 1)) / r, inv_dr = 1 / effective radial spacing (S2AdvectiveCFL, Spherical3DAdvectiveCFL,
 * core/basis.py:6156-6212); u_r / inv_dr may be NULL on the 2-sphere.  `out` must be zero-initialised. */
int db_cfl_max_spherical(const double* u_phi, const double* u_theta, const double* u_r, const double* inv_h, const double* inv_dr,
                         int64_t n_ang, int64_t n_r, double* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif
