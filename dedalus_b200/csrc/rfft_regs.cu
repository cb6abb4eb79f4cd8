// Register-resident real Fourier transforms for the dealiased (3/2-rule) sizes on a strided axis (T1 hot path).
//
// The generic kernel in fft.cu runs log-many shared-memory passes and is bound by instruction issue, not HBM.  Here a
// line of n = 3 * Q * NB grid points is transformed in TWO register stages with ONE shared-memory exchange:
//   * two adjacent real lines (2p, 2p+1) are packed as one complex line z = g1 + i g2 ("two for one"), so every global
//     access is a 16-byte load / store covering both lines, and the real <-> half-complex pre / post processing of the
//     generic kernel collapses to four additions per mode;
//   * length n = NA * NB with NA = 3Q: stage A is a register DFT of size NA, stage B one of size NB; the twiddle between
//     them comes from the plan's exp(-2 pi i j / n) table;
//   * dealias padding is structural: coefficient modes k >= n/3 are zero, which is exactly the middle third of the
//     first radix-3 split of stage A (backward) / the discarded third of its outputs (forward), so that third of the
//     butterflies is never computed and the padded zeros / truncated modes are never touched in memory.
// One CTA = 16 lines (8 complex pairs, 128-byte rows) x the whole line; 48 KB of shared memory (tile height P below).
// Conventions as in fft.cu (reference core/transforms.py:469-509, 537-565): cos / -sin interleaved coefficients,
// forward scaled by 2/n (1/n for k = 0), sin(0) slot zero, Nyquist dropped.
#include "db_common.cuh"
#include <utility>
#include "tw96.inc"

namespace {

struct RegArgs {
    const double* in;
    double* out;
    const double* twn;      // exp(-2 pi i j / n), j < n, interleaved
    int64_t inner;          // stride between line elements (lines are adjacent along inner)
    int32_t M;              // coefficient rows (even, <= 2n/3)
    int32_t deriv;
    double kscale;
    // Blocked row addressing (pencil transposes without pack / unpack kernels, X1): with rpb > 0 row r of outer index o
    // lives at (r / rpb) * blk_stride + (o * rpb + r % rpb) * inner, i.e. the rows are grouped into the per-peer blocks
    // of an all-to-all send buffer (output side) or receive buffer (input side).  rpb = 0: plain (o * rows + r) * inner.
    int32_t in_rpb, out_rpb;
    int64_t in_blk_stride, out_blk_stride;
    // Peer exchange (X1 without a library collective): with out_peers > 0 output block b is not at out + b * out_blk_stride
    // but at out_blk_ptr[b] -- the receive buffer of GPU b, mapped into this process (NVLink peer memory): the transform's
    // own 16-byte stores ARE the all-to-all, overlapped tile by tile with its arithmetic.
    int32_t out_peers;
    double* out_blk_ptr[8];
};

__device__ __forceinline__ int64_t row_offset(int64_t o, int r, int rows, int rpb, int64_t blk_stride, int64_t inner)
{
    if (rpb == 0) return (o * rows + r) * inner;
    const int blk = r / rpb;
    return (int64_t)blk * blk_stride + (o * rpb + (r - blk * rpb)) * inner;
}

// address of output row r of outer index o (plain / blocked / blocked into peer memory)
__device__ __forceinline__ double* out_row_ptr(const RegArgs& a, double* gout, int64_t o, int r, int rows, int64_t inner)
{
    if (a.out_peers > 0) {
        const int blk = r / a.out_rpb;
        return a.out_blk_ptr[blk] + (gout - a.out) + (o * a.out_rpb + (r - blk * a.out_rpb)) * inner;
    }
    return gout + row_offset(o, r, rows, a.out_rpb, a.out_blk_stride, inner);
}

// The forward store's destination in the fused x pass: plain rows only.  Three scalars, so that it stays in registers; a RegArgs
// there would go to local memory (its out_blk_ptr array is indexed at run time).
struct PlainRows {
    const double* twn;
    int64_t inner;
    int32_t M;
};

__device__ __forceinline__ double* out_row_ptr(const PlainRows&, double* gout, int64_t o, int r, int rows, int64_t inner)
{
    return gout + (o * rows + r) * inner;
}

__device__ __forceinline__ double2 cadd2(double2 a, double2 b) { return make_double2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ double2 csub2(double2 a, double2 b) { return make_double2(a.x - b.x, a.y - b.y); }

// a * exp(-/+ 2 pi i NUM / DEN) with the twiddle a compile-time constant (forward: minus sign, INV: plus)
template <int NUM, int DEN, bool INV> __device__ __forceinline__ double2 mul_tw(double2 a)
{
    static_assert(96 % DEN == 0, "twiddle denominators must divide 96");
    constexpr int j = ((NUM % DEN) * (96 / DEN)) % 96;
    if constexpr (j == 0) return a;
    else if constexpr (j == 24) return INV ? make_double2(-a.y, a.x) : make_double2(a.y, -a.x);
    else if constexpr (j == 48) return make_double2(-a.x, -a.y);
    else if constexpr (j == 72) return INV ? make_double2(a.y, -a.x) : make_double2(-a.y, a.x);
    else {
        constexpr double c = tw96_cos(j);
        constexpr double s = INV ? tw96_sin(j) : -tw96_sin(j);
        return make_double2(a.x * c - a.y * s, a.x * s + a.y * c);
    }
}

// natural-order in-register DFT of a power-of-two length (radix-2 decimation in time down to length 4 / 2)
template <int N, bool INV> struct DftP2 {
    template <int... K>
    static __device__ __forceinline__ void combine(double2 (&v)[N], const double2 (&e)[N / 2], const double2 (&o)[N / 2],
                                                   std::integer_sequence<int, K...>)
    {
        ((void)([&] {
            const double2 t = mul_tw<K, N, INV>(o[K]);
            v[K] = cadd2(e[K], t);
            v[K + N / 2] = csub2(e[K], t);
        }()), ...);
    }
    static __device__ __forceinline__ void run(double2 (&v)[N])
    {
        double2 e[N / 2], o[N / 2];
#pragma unroll
        for (int i = 0; i < N / 2; ++i) { e[i] = v[2 * i]; o[i] = v[2 * i + 1]; }
        DftP2<N / 2, INV>::run(e);
        DftP2<N / 2, INV>::run(o);
        combine(v, e, o, std::make_integer_sequence<int, N / 2>{});
    }
};
template <bool INV> struct DftP2<4, INV> {
    static __device__ __forceinline__ void run(double2 (&v)[4])
    {
        const double2 a = cadd2(v[0], v[2]), b = csub2(v[0], v[2]), c = cadd2(v[1], v[3]), d = csub2(v[1], v[3]);
        const double2 jd = INV ? make_double2(-d.y, d.x) : make_double2(d.y, -d.x);
        v[0] = cadd2(a, c); v[2] = csub2(a, c);
        v[1] = cadd2(b, jd); v[3] = csub2(b, jd);
    }
};
template <bool INV> struct DftP2<2, INV> {
    static __device__ __forceinline__ void run(double2 (&v)[2])
    {
        const double2 a = v[0], b = v[1];
        v[0] = cadd2(a, b); v[1] = csub2(a, b);
    }
};

// u[b] *= exp(-/+ 2 pi i b C / NA) for b = 0..Q-1
template <int C, int NA, bool INV, int Q, int... B>
__device__ __forceinline__ void twiddle_row(double2 (&u)[Q], std::integer_sequence<int, B...>)
{
    ((void)(u[B] = mul_tw<(B * C) % NA, NA, INV>(u[B])), ...);
}

__device__ __forceinline__ double2 ldtwn(const double* __restrict__ tw, int j) { return reinterpret_cast<const double2*>(tw)[j]; }
// a * conj(w)
__device__ __forceinline__ double2 cmulc2(double2 a, double2 w) { return make_double2(a.x * w.x + a.y * w.y, a.y * w.x - a.x * w.y); }
__device__ __forceinline__ double2 cmul2(double2 a, double2 w) { return make_double2(a.x * w.x - a.y * w.y, a.x * w.y + a.y * w.x); }

// Tile height: P complex line pairs (2P real lines) per CTA tile.  The kernels take P as a template parameter; the Fourier
// launches below build them at RR_P = 8 only (half-height tiles were measured slower, DESIGN section 4).  The tile's 16 lines are
// what the coverage tests below require of `inner`.
#define RR_P 8
#define RR_LINES (2 * RR_P)

// Persistent CTAs walk the tiles (tile = 2P adjacent lines x the whole line length) with the NEXT tile's input rows in
// flight (16-byte cp.async, L1-bypassing) while the current tile is transformed: two shared-memory buffers of
// n x 16P bytes; the stage A -> stage B exchange reuses the buffer the current tile's input was staged in.
struct TileWalk {
    int64_t tiles_per_outer, total;
};

// stage `rows` rows of 2P doubles (row stride `inner`) into buf[row][2P]
template <int P>
__device__ __forceinline__ void stage_rows(double* buf, const double* __restrict__ src, int64_t o, int rows, int rpb,
                                           int64_t blk_stride, int64_t inner)
{
    // src already points at the tile's first column; row r of outer index o is at row_offset(...)
    for (int idx = threadIdx.x; idx < rows * P; idx += blockDim.x) {
        const int row = (unsigned)idx / P, seg = (unsigned)idx % P;
        db_cp_async16(buf + row * (2 * P) + seg * 2, src + row_offset(o, row, rows, rpb, blk_stride, inner) + seg * 2);
    }
}

// Thread layout.  Both register stages are split so that no thread holds more than max(Q, NB/2) complex values:
//   stage A (size NA = 3Q): thread (c, n2, p) computes the Q outputs k1 = c + 3 kb of the radix-3 residue c
//   stage B (size NB):      thread (h, k1, p) computes the NB/2 outputs k2 = 2 m + h (first radix-2 split, DIF)
// (forward: the same two splits in the opposite order).  3 NB P threads work in stage A and 6 Q P in stage B: 384 = 384
// at n = 384 and P = 8, at ~80 registers, so two CTAs (24 warps) are resident per SM and every warp works in both stages.
// minb() keeps 768 threads per SM (the same register budget per thread at any P) where shared memory allows.  The forward and
// the derivative backward transforms of lines of 192 or more points need more than the ~80 registers that leaves: they spill
// (320 and 460 bytes at n = 384) and run at about half the bandwidth of the plain backward.  minb(true) gives them the whole
// register file of one CTA (no spills in the forward, 88 bytes in the backward), which is faster despite the single CTA per SM;
// the launches size their grids from the resulting occupancy.
template <int Q, int NB, int P> struct RegGeom {
    static constexpr int NA = 3 * Q, N = NA * NB;
    static constexpr int TA = 3 * NB * P, TB = 6 * Q * P;
    static constexpr int THREADS = TA > TB ? TA : TB;
    static constexpr int minb(bool full_regs = false)
    {
        const int fit = (int)((226 * 1024) / (2 * N * P * 16 + 1024));
        return full_regs && N >= 192 ? 1 : fit < 1 ? 1 : (fit < 16 / P ? fit : 16 / P);
    }
};

template <bool INV, int N, int... M>
__device__ __forceinline__ void twiddle_odd_half(double2 (&o)[N], std::integer_sequence<int, M...>)
{
    ((void)(o[M] = mul_tw<M, 2 * N, INV>(o[M])), ...);
}

// forward stage 2, residue C of the outputs: t[b] = sum_a' W3^(a' C) B[Q a' + b], times W_NA^(b C)
template <int C, int Q>
__device__ __forceinline__ void residue_gather(double2 (&u)[Q], const double2* src, int stride)
{
#pragma unroll
    for (int b = 0; b < Q; ++b) {
        const double2 b0 = src[b * stride], b1 = src[(Q + b) * stride], b2 = src[(2 * Q + b) * stride];
        u[b] = cadd2(b0, cadd2(mul_tw<C % 3, 3, false>(b1), mul_tw<(2 * C) % 3, 3, false>(b2)));
    }
    twiddle_row<C, 3 * Q, false>(u, std::make_integer_sequence<int, Q>{});
}

// ---------------------------------------------------------------------------------------------------------
// The register stages of the x passes, shared by k_rbwd_regs / k_rfwd_regs and the fused k_rfft_x_products.
// Roles of thread (p, r): p = line pair of the tile, r = threadIdx.x / P (see RegGeom).
// ---------------------------------------------------------------------------------------------------------

// backward, load + stage A: spectrum of the staged coefficient rows `in` ([M][P] double2: row 2k = re, 2k+1 = im of mode k
// for both lines of every pair) with (i k kscale)^deriv applied, then this thread's residue of the size-NA DFT (threads r < 3 NB)
template <int Q, int NB, int P, bool DERIV>
__device__ __forceinline__ void rbwd_load_a(const double2* in, int p, int r, int M, int deriv_, double kscale, double2 (&u)[Q])
{
    const int Kmax = (M - 1) / 2;
    const int deriv = DERIV ? deriv_ : 0;
    // (i k kscale)^deriv = (ur + i ui) (k kscale)^deriv
    const double ur = ((deriv & 3) == 0) ? 1.0 : ((deriv & 3) == 2) ? -1.0 : 0.0;
    const double ui = ((deriv & 3) == 1) ? 1.0 : ((deriv & 3) == 3) ? -1.0 : 0.0;
    const int n2 = r % NB, c = r / NB;
    // Z_k = X1_k + i X2_k (k <= Kmax), Z_{n-k} = conj X1_k + i conj X2_k, X_k = (c_2k + i c_2k+1) / 2, X_0 = c_0
    auto spec = [&](int k, bool mirrored) -> double2 {
        if (k > Kmax) return make_double2(0.0, 0.0);
        const double2 R = in[(2 * k) * P + p];                      // (re line 1, re line 2)
        if (k == 0) return DERIV ? make_double2(0.0, 0.0) : R;
        const double2 I = in[(2 * k + 1) * P + p];                  // (im line 1, im line 2)
        if (DERIV) {
            const double ks = kscale * k, ks2 = ks * ks;
            const double f = 0.5 * ((deriv == 1) ? ks : (deriv == 2) ? ks2 : (deriv == 3) ? ks2 * ks : ks2 * ks2);
            const double mr = ur * f, mi = ui * f;
            const double2 R2 = make_double2(mr * R.x - mi * I.x, mr * R.y - mi * I.y);
            const double2 I2 = make_double2(mi * R.x + mr * I.x, mi * R.y + mr * I.y);
            return mirrored ? make_double2(R2.x + I2.y, R2.y - I2.x) : make_double2(R2.x - I2.y, I2.x + R2.y);
        }
        return mirrored ? make_double2(0.5 * (R.x + I.y), 0.5 * (R.y - I.x)) : make_double2(0.5 * (R.x - I.y), 0.5 * (I.x + R.y));
    };
    // stage A: size-NA DFT over n1 = Q a + b with the a = 1 third identically zero; this thread's residue c:
    // u[b] = Z[NB b + n2] + W3^(2c) Z[NB (2Q + b) + n2], times W_NA^(b c), each pair of modes combined as soon as it is loaded
    // (the spectrum is never held in registers as a whole)
    double2 lo[Q], hi[Q];
#pragma unroll
    for (int b = 0; b < Q; ++b) {
        lo[b] = spec(NB * b + n2, false);
        hi[b] = spec(NB * (Q - b) - n2, true);
    }
    auto combine = [&](auto CC) {
        constexpr int C = decltype(CC)::value;
#pragma unroll
        for (int b = 0; b < Q; ++b) u[b] = cadd2(lo[b], mul_tw<(2 * C) % 3, 3, true>(hi[b]));
        twiddle_row<C, 3 * Q, true>(u, std::make_integer_sequence<int, Q>{});
    };
    if (c == 0) combine(std::integral_constant<int, 0>{});
    else if (c == 1) combine(std::integral_constant<int, 1>{});
    else combine(std::integral_constant<int, 2>{});
}

// backward, end of stage A: radix-2 part and twiddle, stored to the exchange buffer ([N][P] double2, threads r < 3 NB)
template <int Q, int NB, int P>
__device__ __forceinline__ void rbwd_exchange_a(double2 (&u)[Q], double2* xch, const double* __restrict__ tw, int p, int r)
{
    const int n2 = r % NB, c = r / NB;
    DftP2<Q, true>::run(u);
    double2* dst = xch + n2 * P + p;
#pragma unroll
    for (int kb = 0; kb < Q; ++kb) {
        const int kk = 3 * kb + c;                         // output k1
        dst[kk * NB * P] = cmulc2(u[kb], ldtwn(tw, n2 * kk));
    }
}

// backward stage B (threads r < 6 Q): size-NB DFT over n2 for fixed k1 = r % NA, outputs k2 = 2 m + h (h = r / NA), so v[m] is
// the pair's grid value at j = k1 + NA (2 m + h)
template <int Q, int NB, int P>
__device__ __forceinline__ void rbwd_stage_b(const double2* xch, int p, int r, double2 (&v)[NB / 2])
{
    constexpr int NA = 3 * Q, H = NB / 2;
    const int k1 = r % NA, h = r / NA;
    const double2* src = xch + (k1 * NB) * P + p;
    if (h == 0) {
#pragma unroll
        for (int m = 0; m < H; ++m) v[m] = cadd2(src[m * P], src[(m + H) * P]);
    } else {
#pragma unroll
        for (int m = 0; m < H; ++m) v[m] = csub2(src[m * P], src[(m + H) * P]);
        twiddle_odd_half<true>(v, std::make_integer_sequence<int, H>{});
    }
    DftP2<H, true>::run(v);
}

// forward stage 1 load (threads r < 6 Q): first radix-2 split (DIF) of the size-NB DFT over j2 for fixed j1 = r % NA of the staged
// grid rows `in` ([N][P] double2, grid index j = j1 + NA j2)
template <int Q, int NB, int P>
__device__ __forceinline__ void rfwd_load_1(const double2* in, int p, int r, double2 (&v)[NB / 2])
{
    constexpr int NA = 3 * Q, H = NB / 2;
    const int j1 = r % NA, h = r / NA;
    const double2* src = in + j1 * P + p;
    if (h == 0) {
#pragma unroll
        for (int m = 0; m < H; ++m) v[m] = cadd2(src[(NA * m) * P], src[(NA * (m + H)) * P]);
    } else {
#pragma unroll
        for (int m = 0; m < H; ++m) v[m] = csub2(src[(NA * m) * P], src[(NA * (m + H)) * P]);
        twiddle_odd_half<false>(v, std::make_integer_sequence<int, H>{});
    }
}

// forward, end of stage 1: the rest of the size-NB DFT and the twiddle, stored to the exchange buffer
template <int Q, int NB, int P>
__device__ __forceinline__ void rfwd_exchange_1(double2 (&v)[NB / 2], double2* xch, const double* __restrict__ tw, int p, int r)
{
    constexpr int NA = 3 * Q, H = NB / 2;
    const int j1 = r % NA, h = r / NA;
    DftP2<H, false>::run(v);
    double2* dst = xch + (j1 * NB + h) * P + p;
#pragma unroll
    for (int m = 0; m < H; ++m) {
        const int kk = 2 * m + h;                          // output k2
        dst[(2 * m) * P] = (kk == 0) ? v[m] : cmul2(v[m], ldtwn(tw, j1 * kk));
    }
}

// forward stage 2 (threads r < 3 NB): size-NA DFT over j1 = Q a' + b for fixed k2 = r % NB; this thread's output residue
// c = r / NB: z[kb] is mode k1 = c + 3 kb
template <int Q, int NB, int P>
__device__ __forceinline__ void rfwd_stage_2(const double2* xch, int p, int r, double2 (&z)[Q])
{
    const int k2 = r % NB, c = r / NB;
    const double2* src = xch + k2 * P + p;
    if (c == 0) residue_gather<0, Q>(z, src, NB * P);
    else if (c == 1) residue_gather<1, Q>(z, src, NB * P);
    else residue_gather<2, Q>(z, src, NB * P);
    DftP2<Q, false>::run(z);
}

// forward: park the high third (k1 >= 2Q) as Zhi[k1 - 2Q][k2] for the mirror partners
template <int Q, int NB, int P>
__device__ __forceinline__ void rfwd_park(const double2 (&z)[Q], double2* xch, int p, int r)
{
    const int k2 = r % NB, c = r / NB;
    double2* dst = xch + k2 * P + p;
#pragma unroll
    for (int kb = 0; kb < Q; ++kb) {
        const int kk = 3 * kb + c;
        if (kk >= 2 * Q) dst[(kk - 2 * Q) * NB * P] = z[kb];
    }
}

// forward: the two real lines' cos / -sin coefficients of every mode k <= Kmax this thread owns, scaled, stored to rows 2k, 2k+1
// (Args: RegArgs or PlainRows)
template <int Q, int NB, int P, class Args>
__device__ __forceinline__ void rfwd_store(const double2 (&z)[Q], const double2* xch, int p, int r, const Args& a, double* gout,
                                           int64_t o)
{
    constexpr int N = 3 * Q * NB;
    const int k2 = r % NB, c = r / NB;
    const int M = a.M, Kmax = (a.M - 1) / 2;
    const int64_t inner = a.inner;
    // Z_{n-k} for k = NB k1 + k2 sits at Zhi[(Q - 1 - k1), NB - k2] for k2 > 0, Zhi[Q - k1, 0] for k2 = 0
    const double sc = 1.0 / N;
    const int k2p = (k2 == 0) ? 0 : NB - k2;
    const double2* src = xch + k2p * P + p;
#pragma unroll
    for (int kb = 0; kb < Q; ++kb) {
        const int kk = 3 * kb + c;                         // k1
        const int k = NB * kk + k2;
        if (kk >= Q || k > Kmax) continue;
        double* row = out_row_ptr(a, gout, o, 2 * k, M, inner);
        double* row1 = out_row_ptr(a, gout, o, 2 * k + 1, M, inner);
        const double2 za = z[kb];
        if (k == 0) {
            *reinterpret_cast<double2*>(row) = make_double2(za.x * sc, za.y * sc);
            *reinterpret_cast<double2*>(row1) = make_double2(0.0, 0.0);
        } else {
            const int kbp = (k2 == 0) ? Q - kk : Q - 1 - kk;
            const double2 zb = src[kbp * NB * P];
            *reinterpret_cast<double2*>(row) = make_double2((za.x + zb.x) * sc, (za.y + zb.y) * sc);
            *reinterpret_cast<double2*>(row1) = make_double2((za.y - zb.y) * sc, (zb.x - za.x) * sc);
        }
    }
}

struct OutCol { double* g; int64_t o; };       // a pair's column in the output rows, outer index

// the whole forward transform of the grid tile staged in `buf` ([N][P] double2), which is also its exchange buffer; every
// thread of the CTA calls it (it contains barriers), and `buf` may be overwritten once the caller has passed a barrier after it.
// dest() -> (this pair's column in the output rows, outer index) is evaluated only at the store.
template <int Q, int NB, int P, class Args, class Dest>
__device__ __forceinline__ void rfwd_tile(double2* buf, int p, int r, const Args& a, Dest dest)
{
    constexpr int NA = 3 * Q, H = NB / 2;
    const bool in_1 = r < 2 * NA, in_2 = r < 3 * NB;
    double2 v[H];
    if (in_1) rfwd_load_1<Q, NB, P>(buf, p, r, v);
    __syncthreads();                                           // inputs are consumed: reuse `buf` as exchange
    if (in_1) rfwd_exchange_1<Q, NB, P>(v, buf, a.twn, p, r);
    __syncthreads();
    double2 z[Q];
    if (in_2) rfwd_stage_2<Q, NB, P>(buf, p, r, z);
    __syncthreads();
    if (in_2) rfwd_park<Q, NB, P>(z, buf, p, r);
    __syncthreads();
    if (in_2) {
        const auto d = dest();
        rfwd_store<Q, NB, P>(z, buf, p, r, a, d.g, d.o);
    }
}

// ---------------------------------------------------------------------------------------------------------
// backward: coefficients (M rows) -> grid (n rows)
// ---------------------------------------------------------------------------------------------------------
template <int Q, int NB, int P, bool DERIV>
__global__ void __launch_bounds__((RegGeom<Q, NB, P>::THREADS), (RegGeom<Q, NB, P>::minb(DERIV)))
k_rbwd_regs(RegArgs a, TileWalk tw_)
{
    using G = RegGeom<Q, NB, P>;
    constexpr int NA = G::NA, N = G::N, H = NB / 2;
    DB_SMEM(double2, sm);                                   // 2 buffers of [N][P] double2
    const int p = threadIdx.x % P, r = threadIdx.x / P;
    const int64_t inner = a.inner;
    const int M = a.M;
    auto stage_tile = [&](double2* buf, int64_t t) { const int64_t o = t / tw_.tiles_per_outer, xt = t - o * tw_.tiles_per_outer;
        stage_rows<P>(reinterpret_cast<double*>(buf), a.in + xt * (2 * P), o, M, a.in_rpb, a.in_blk_stride, inner); };
    const bool in_a = r < 3 * NB, in_b = r < 2 * NA;
    const int k1 = r % NA, h = r / NA;                       // stage B role
    int64_t t = blockIdx.x;
    int cur = 0;
    if (t < tw_.total) stage_tile(sm, t);
    db_cp_commit();
    for (; t < tw_.total; t += gridDim.x, cur ^= 1) {
        double2* in = sm + cur * (N * P);
        const int64_t tn = t + gridDim.x;
        if (tn < tw_.total) stage_tile(sm + (cur ^ 1) * (N * P), tn);
        db_cp_commit();
        db_cp_wait<1>();
        __syncthreads();
        double2 u[Q];
        if (in_a) rbwd_load_a<Q, NB, P, DERIV>(in, p, r, M, a.deriv, a.kscale, u);
        __syncthreads();                                           // every input value is consumed: reuse `in` as exchange
        if (in_a) rbwd_exchange_a<Q, NB, P>(u, in, a.twn, p, r);
        __syncthreads();
        if (in_b) {
            double2 v[H];
            rbwd_stage_b<Q, NB, P>(in, p, r, v);
            const int64_t o = t / tw_.tiles_per_outer, xt = t - o * tw_.tiles_per_outer;
            double* __restrict__ gout = a.out + xt * (2 * P) + 2 * p;
#pragma unroll
            for (int m = 0; m < H; ++m)
                *reinterpret_cast<double2*>(out_row_ptr(a, gout, o, k1 + NA * (2 * m + h), N, inner)) = v[m];
        }
        __syncthreads();                                           // exchange reads done before the next prefetch lands here
    }
    db_cp_wait<0>();
}

// ---------------------------------------------------------------------------------------------------------
// forward: grid (n rows) -> coefficients (M rows)
// ---------------------------------------------------------------------------------------------------------
template <int Q, int NB, int P>
__global__ void __launch_bounds__((RegGeom<Q, NB, P>::THREADS), (RegGeom<Q, NB, P>::minb(true)))
k_rfwd_regs(RegArgs a, TileWalk tw_)
{
    using G = RegGeom<Q, NB, P>;
    constexpr int N = G::N;
    DB_SMEM(double2, sm);                                   // 2 buffers of [N][P] double2
    const int p = threadIdx.x % P, r = threadIdx.x / P;
    const int64_t inner = a.inner;
    auto stage_tile = [&](double2* buf, int64_t t) { const int64_t o = t / tw_.tiles_per_outer, xt = t - o * tw_.tiles_per_outer;
        stage_rows<P>(reinterpret_cast<double*>(buf), a.in + xt * (2 * P), o, N, a.in_rpb, a.in_blk_stride, inner); };
    int64_t t = blockIdx.x;
    int cur = 0;
    if (t < tw_.total) stage_tile(sm, t);
    db_cp_commit();
    for (; t < tw_.total; t += gridDim.x, cur ^= 1) {
        double2* in = sm + cur * (N * P);
        const int64_t tn = t + gridDim.x;
        if (tn < tw_.total) stage_tile(sm + (cur ^ 1) * (N * P), tn);
        db_cp_commit();
        db_cp_wait<1>();
        __syncthreads();
        rfwd_tile<Q, NB, P>(in, p, r, a, [&] {
            const int64_t o = t / tw_.tiles_per_outer, xt = t - o * tw_.tiles_per_outer;
            return OutCol{a.out + xt * (2 * P) + 2 * p, o};
        });
        __syncthreads();
    }
    db_cp_wait<0>();
}

// ---------------------------------------------------------------------------------------------------------
// Fused x pass of a right-hand side: backward x transforms of the inputs -> quadratic products -> forward x transforms of the
// outputs, one tile (16 lines x the whole x line) at a time, so that no grid array goes through global memory.
//
// A tile walks the host-built schedule `items`:
//   * held items transform an input that appears in several terms (the velocity components of u.grad(u), u.grad(b)) and keep
//     this thread's grid values in shared memory (a slot private to the thread, so no barrier guards it);
//   * term items add coef * a * b (or coef * a) to the output's accumulator, exactly as k_pointwise_pairs does; a term with a
//     streamed factor first transforms that input (with its x derivative), and its grid values are used straight from registers;
//   * after the last term of an output the accumulator goes through shared memory into the forward transform, whose coefficient
//     rows are stored to the output array.
// Every thread accumulates at the grid points it owns after backward stage B, so products need no exchange.  The coefficient
// rows of the next transform are in flight (cp.async) from the moment the current ones are in registers (after stage A) until
// the next item starts: through stage B, the products and, after an output's last term, its forward transform.
//
// Shared memory at n = 384, M = 256, three held factors: exchange [N][P] 48 KB + staging [M][P] 32 KB + 3 held tiles 144 KB =
// 224 KB, one CTA of 384 threads per SM.  Holding a factor in registers instead (32 more per thread, for a second staging slot)
// takes the kernel past the 168 registers a 384-thread CTA can have and makes it spill.  That shared-memory carve-out leaves the
// SM about 30 KB of L1, so local memory is expensive here: the forward store gets a destination that stays in registers
// (PlainRows), and the thread roles are re-derived per item (see below).
// ---------------------------------------------------------------------------------------------------------
#define XP_STREAM 3             // factor code of the streamed input (0..2: held factors, -1: none)

struct XProdArgs {
    const double* in;           // stack of level arrays: input s at in + s * in_stride, rows M x inner
    double* out;                // outputs: o at out + o * out_stride, rows M x inner
    const double* twn;
    int64_t inner, in_stride, out_stride;
    int32_t M;
    double kscale;
    const db_xprod_item* items;
    int32_t n_items;
    const int32_t* loads;       // src of every item with src >= 0, in item order
    int32_t n_loads;
};

// threadIdx.x (< THREADS) read anew at every call (volatile asm), so that nothing derived from it can be hoisted out of the loop
// it is read in; the bound keeps the compiler's knowledge of which thread roles exist
template <int THREADS> __device__ __forceinline__ int opaque_tid()
{
#ifdef DB_EMU
    return (int)threadIdx.x;
#else
    unsigned t;
    asm volatile("mov.u32 %0, %%tid.x;" : "=r"(t));
    __builtin_assume(t < THREADS);
    return (int)t;
#endif
}

// MINB: the register budget per thread (168 at n = 384) is the same at every tile height: 8 / P CTAs of 48 P threads per SM
template <int Q, int NB, int P> struct XpGeom {
    static constexpr int N = 3 * Q * NB, THREADS = RegGeom<Q, NB, P>::THREADS, H = NB / 2, MINB = 8 / P;
    static size_t smem(int M, int n_held)
    {
        return sizeof(double2) * ((size_t)N * P + (size_t)M * P + (size_t)n_held * H * THREADS);
    }
};

template <int Q, int NB, int P>
__global__ void __launch_bounds__((XpGeom<Q, NB, P>::THREADS), (XpGeom<Q, NB, P>::MINB))
k_rfft_x_products(XProdArgs a, int64_t total)
{
    using G = RegGeom<Q, NB, P>;
    constexpr int NA = G::NA, N = G::N, H = NB / 2, THREADS = G::THREADS;
    DB_SMEM(double2, sm);
    const int M = a.M;
    double2* X = sm;                                       // [N][P] exchange / forward staging
    double2* stg = X + N * P;                              // [M][P] coefficient rows of the next transform
    double2* hs = stg + M * P;                             // held factors: [H][THREADS] each, private to their thread
    const int64_t inner = a.inner;
    const PlainRows fa{a.twn, inner, M};
    // load sequence of this CTA: for each of its tiles, every entry of a.loads
    int64_t ld_t = blockIdx.x;
    int ld_k = 0;
    auto issue = [&] {
        if (ld_t < total) {
            stage_rows<P>(reinterpret_cast<double*>(stg), a.in + a.loads[ld_k] * a.in_stride + ld_t * (2 * P), 0, M, 0, 0, inner);
            if (++ld_k == a.n_loads) { ld_k = 0; ld_t += gridDim.x; }
        }
    };
    issue();
    db_cp_commit();
    double2 acc[H];
#pragma unroll
    for (int m = 0; m < H; ++m) acc[m] = make_double2(0.0, 0.0);
    for (int64_t t = blockIdx.x; t < total; t += gridDim.x) {
        for (int i = 0; i < a.n_items; ++i) {
            const db_xprod_item* itp = a.items + i;
            // Thread roles per item: derived once per kernel, the shared-memory and twiddle addresses and derivative factors of
            // every unrolled stage would be hoisted out of the loop, live across all its transforms, and spill.
            const int tid = opaque_tid<THREADS>(), p = tid % P, r = tid / P;
            const bool in_a = r < 3 * NB, in_b = r < 2 * NA;
            const int k1 = r % NA, h = r / NA;
            double2 v[H];
            if (itp->src >= 0) {
                db_cp_wait<0>();
                __syncthreads();                           // this input's rows have landed for every thread; X is free
                double2 u[Q];
                if (in_a) {
                    const int deriv = itp->deriv;
                    if (deriv == 0) rbwd_load_a<Q, NB, P, false>(stg, p, r, M, 0, a.kscale, u);
                    else rbwd_load_a<Q, NB, P, true>(stg, p, r, M, deriv, a.kscale, u);
                    rbwd_exchange_a<Q, NB, P>(u, X, a.twn, p, r);
                }
                __syncthreads();                           // staging consumed, exchange written
                issue();
                db_cp_commit();
                if (in_b) rbwd_stage_b<Q, NB, P>(X, p, r, v);
            }
            const db_xprod_item it = *itp;                 // (read after the transforms, and again at the store: not live across them)
            if (in_b) {
                auto factor = [&](int f, int m) -> double2 {
                    return f == XP_STREAM ? v[m] : hs[(f * H + m) * THREADS + tid];
                };
                if (it.flags & DB_XPROD_HELD) {
#pragma unroll
                    for (int m = 0; m < H; ++m) hs[(it.a * H + m) * THREADS + tid] = v[m];
                } else {
#pragma unroll
                    for (int m = 0; m < H; ++m) {
                        const double2 va = factor(it.a, m);
                        const double p0 = it.coef * va.x, p1 = it.coef * va.y;
                        if (it.b >= 0) {
                            const double2 vb = factor(it.b, m);
                            acc[m].x = fma(p0, vb.x, acc[m].x); acc[m].y = fma(p1, vb.y, acc[m].y);
                        } else { acc[m].x += p0; acc[m].y += p1; }
                    }
                }
            }
            if (it.flags & DB_XPROD_LAST) {
                __syncthreads();                           // stage B reads of X are done
                if (in_b) {
#pragma unroll
                    for (int m = 0; m < H; ++m) { X[(k1 + NA * (2 * m + h)) * P + p] = acc[m]; acc[m] = make_double2(0.0, 0.0); }
                }
                __syncthreads();
                rfwd_tile<Q, NB, P>(X, p, r, fa, [&] { return OutCol{a.out + itp->out * a.out_stride + t * (2 * P) + 2 * p, 0}; });
                __syncthreads();
            }
        }
    }
    db_cp_wait<0>();
}

// =========================================================================================================
// Chebyshev (DCT-II / DCT-III) along CONTIGUOUS lines with the same two register stages (T2 on the benchmark path).
// A tile is 16 adjacent lines = one contiguous block of global memory; lines are staged in shared memory as
// X[line][n + 2] (the +2 spreads line pairs over the banks), two adjacent lines form one complex line, and the DCT runs
// through the full-length complex FFT of the even/odd reordered sequence (Makhoul): v[m] = g[2m] (m < n/2),
// v[m] = g[2(n-1-m)+1] otherwise;
//   backward: Z_k = w_k ((a1 + b2) + i (a2 - b1)), a = c^_k, b = c^_{n-k}, w_k = exp(i pi k / 2n), c^ = scaled, sign-
//             flipped coefficients (zero beyond the coefficient size);  v1 + i v2 = IDFT_n(Z)
//   forward : Z = DFT_n(v1 + i v2);  C1_k = s_k Re(q^k (Z_k + conj Z_{n-k})),  C2_k = s_k Re(q^k (Z_k - conj Z_{n-k}) / i),
//             q = conj w; truncation to the coefficient size and the banded ultraspherical conversion are applied while
//             the coefficient lines are still in shared memory.
// Conventions as fft.cu K_CHFWD / K_CHBWD (reference core/transforms.py:715-746, 771-902).
// =========================================================================================================
struct ChebArgs {
    const double* in;
    double* out;
    const double* twn;      // exp(-2 pi i j / n)
    const double* twq;      // exp(-i pi k / (2 n))
    const double* diags;    // forward: conversion diagonals [nd][M]
    const double* pre;      // backward: derivative diagonals [npre][M] applied first (npre <= 3), or null
    const double* sol2;     // backward: [2][M] reciprocal diagonal and second super-diagonal of the back-conversion, or null
    int64_t lines;
    int32_t M;              // coefficient size (even, <= n)
    int32_t nd;
    int32_t npre;
};

// Tile height.  The z kernels are one tile per CTA with full-CTA barriers between their phases, i.e. latency-bound at
// 2 CTAs / SM (long-scoreboard stalls): P = line pairs per tile is a template parameter so that lines of 192 points or more
// take smaller tiles (P = 4: 8 lines, 192 threads, 49 KB at n = 384 -> 4 CTAs / SM in different phases) that hide it;
// shorter lines keep P = 8 (launch_cheb).
template <int Q, int NB, int P> struct ChGeom {
    static_assert(P == 8 || P == 4, "Chebyshev tiles are 8 or 4 line pairs high");
    static constexpr int NA = 3 * Q, N = NA * NB, LINES = 2 * P;
    static constexpr int TA = 3 * NB * P, TB = 6 * Q * P;
    static constexpr int THREADS = TA > TB ? TA : TB;
    static constexpr int LOGP = P == 8 ? 3 : 2;
    static constexpr size_t SMEM = (size_t)LINES * (N + 2) * sizeof(double) + (size_t)N * P * sizeof(double2);
    static constexpr int MINB = (int)((226 * 1024) / (SMEM + 1024)) > 8 ? 8 : ((int)((226 * 1024) / (SMEM + 1024)) < 1 ? 1 : (int)((226 * 1024) / (SMEM + 1024)));
};

template <int Q, int NB, int P>
__global__ void __launch_bounds__((ChGeom<Q, NB, P>::THREADS), (ChGeom<Q, NB, P>::MINB))
k_chbwd_regs(ChebArgs a)
{
    using G = ChGeom<Q, NB, P>;
    constexpr int NA = G::NA, N = G::N, H = NB / 2, LX = N + 2, CH_LINES = G::LINES;
    DB_SMEM(double, X);                                      // [16][LX] doubles, then Y = [N][P] double2
    double2* Y = reinterpret_cast<double2*>(X + CH_LINES * LX);
    const int tid = threadIdx.x, nthreads = blockDim.x;
    const int M = a.M;
    const int64_t l0 = (int64_t)blockIdx.x * CH_LINES;
    const int nl = (a.lines - l0 < CH_LINES) ? (int)(a.lines - l0) : CH_LINES;
    // ---- stage the coefficient lines (16-byte chunks); missing lines of a partial tile are zero
    {
        // one warp per line at a time, lanes along the line (16-byte chunks): no index division
        const int cpl = M / 2, lane = tid & 31, nw = nthreads >> 5;
        for (int l = tid >> 5; l < CH_LINES; l += nw) {
            double* dst = X + l * LX;
            if (l < nl) {
                const double* src = a.in + (l0 + l) * M;
                for (int ch = lane; ch < cpl; ch += 32) db_cp_async16(dst + 2 * ch, src + 2 * ch);
            } else {
                for (int ch = lane; ch < cpl; ch += 32) { dst[2 * ch] = 0.0; dst[2 * ch + 1] = 0.0; }
            }
        }
        db_cp_commit();
        db_cp_wait<0>();
    }
    __syncthreads();
    if (a.sol2 != nullptr) {
        // derivative + ultraspherical back-conversion in place on the staged lines (same suffix scan as k_band_scan2 in
        // fft.cu: x_i = r_i (t_i - u_i x_{i+2}), t = banded pre-apply of the coefficients), one warp per line
        const int lane = tid & 31, w = tid >> 5, nw = nthreads >> 5;
        const double* __restrict__ pre = a.pre;
        const double* __restrict__ sol = a.sol2;
        const int npre = a.npre, rounds = (M + 63) / 64;
        for (int l = w; l < CH_LINES; l += nw) {
            double* xl = X + l * LX;
            double carry0 = 0.0, carry1 = 0.0, nx0 = 0.0, nx1 = 0.0;     // nx: ORIGINAL c[i0+2], c[i0+3] of the round above
            for (int q = rounds - 1; q >= 0; --q) {
                const int i0 = 2 * (32 * q + lane);
                const double c0 = (i0 < M) ? xl[i0] : 0.0, c1 = (i0 + 1 < M) ? xl[i0 + 1] : 0.0;
                double c2 = __shfl_down_sync(0xffffffffu, c0, 1), c3 = __shfl_down_sync(0xffffffffu, c1, 1);
                if (lane == 31) { c2 = nx0; c3 = nx1; }
                nx0 = __shfl_sync(0xffffffffu, c0, 0); nx1 = __shfl_sync(0xffffffffu, c1, 0);
                double t0 = c0, t1 = c1;
                if (npre > 0) {
                    t0 = 0.0; t1 = 0.0;
                    if (i0 < M) {
                        t0 = pre[i0] * c0;
                        if (npre > 1) t0 = fma(pre[M + i0], c1, t0);
                        if (npre > 2) t0 = fma(pre[2 * M + i0], c2, t0);
                    }
                    if (i0 + 1 < M) {
                        t1 = pre[i0 + 1] * c1;
                        if (npre > 1) t1 = fma(pre[M + i0 + 1], c2, t1);
                        if (npre > 2) t1 = fma(pre[2 * M + i0 + 1], c3, t1);
                    }
                }
                double A0 = 0.0, B0 = 0.0, A1 = 0.0, B1 = 0.0;
                if (i0 < M) { const double rr = sol[i0]; B0 = rr * t0; A0 = (i0 + 2 < M) ? -rr * sol[M + i0] : 0.0; }
                if (i0 + 1 < M) { const double rr = sol[i0 + 1]; B1 = rr * t1; A1 = (i0 + 3 < M) ? -rr * sol[M + i0 + 1] : 0.0; }
#pragma unroll
                for (int off = 1; off < 32; off <<= 1) {
                    const double a0 = __shfl_down_sync(0xffffffffu, A0, off), b0 = __shfl_down_sync(0xffffffffu, B0, off);
                    const double a1 = __shfl_down_sync(0xffffffffu, A1, off), b1 = __shfl_down_sync(0xffffffffu, B1, off);
                    if (lane + off < 32) { B0 = fma(A0, b0, B0); A0 *= a0; B1 = fma(A1, b1, B1); A1 *= a1; }
                }
                const double x0 = fma(A0, carry0, B0), x1 = fma(A1, carry1, B1);
                if (i0 < M) xl[i0] = x0;
                if (i0 + 1 < M) xl[i0 + 1] = x1;
                carry0 = __shfl_sync(0xffffffffu, x0, 0); carry1 = __shfl_sync(0xffffffffu, x1, 0);
            }
        }
        __syncthreads();
    }
    // ---- spectrum of the packed line pairs: Y[k][p] = Z_k
    {
        const double c0 = 0.56418958354775628694807945156077;     // 1/sqrt(pi)
        const double c1 = 0.39894228040143267793994605993438;     // 1/sqrt(2 pi)
        // warp task = (block of 8 modes, half of the line pairs); lanes = 4 pairs x 8 modes (bank-friendly on both sides)
        const int lane = tid & 31, w = tid >> 5, nw = nthreads >> 5;
        constexpr int PL = P < 4 ? P : 4, KL = 32 / PL, PH = P / PL;       // lanes = PL pairs x KL modes; PH warp tasks per mode block
        const int kk = lane / PL;
        for (int wt = w; wt < PH * ((N + KL - 1) / KL); wt += nw) {
            const int k = (wt / PH) * KL + kk, pp = (lane % PL) + PL * (wt % PH);
            if (k >= N) continue;
            const double* x1 = X + (2 * pp) * LX;
            const double* x2 = x1 + LX;
            const int kb = N - k;
            const double sa = ((k == 0) ? c0 : c1) * ((k & 1) ? -1.0 : 1.0);
            const double sb = c1 * ((kb & 1) ? -1.0 : 1.0);
            const bool ha = k < M, hb = (k > 0) && (kb < M);
            const double a1 = ha ? x1[k] * sa : 0.0, a2 = ha ? x2[k] * sa : 0.0;
            const double b1 = hb ? x1[kb] * sb : 0.0, b2 = hb ? x2[kb] * sb : 0.0;
            const double2 wq = ldtwn(a.twq, k);              // exp(-i pi k / 2n): conj of w_k
            Y[k * P + pp] = cmulc2(make_double2(a1 + b2, a2 - b1), wq);
        }
    }
    __syncthreads();
    const int p = tid & (P - 1), r = tid >> G::LOGP;
    const bool in_a = r < 3 * NB, in_b = r < 2 * NA;
    const int n2 = r % NB, c = r / NB;
    const int k1 = r % NA, h = r / NA;
    const double* __restrict__ tw = a.twn;
    double2 u[Q];
    if (in_a) {
        const double2* src = Y + n2 * P + p;
        // stage A residue c: u[b] = sum_a W3^(a c) Z[NB (Q a + b) + n2], times W_NA^(b c)      (inverse signs)
        auto gather = [&](auto CC) {
            constexpr int C = decltype(CC)::value;
#pragma unroll
            for (int b = 0; b < Q; ++b) {
                const double2 z0 = src[(NB * b) * P], z1 = src[(NB * (Q + b)) * P], z2 = src[(NB * (2 * Q + b)) * P];
                u[b] = cadd2(z0, cadd2(mul_tw<C % 3, 3, true>(z1), mul_tw<(2 * C) % 3, 3, true>(z2)));
            }
            twiddle_row<C, NA, true>(u, std::make_integer_sequence<int, Q>{});
        };
        if (c == 0) gather(std::integral_constant<int, 0>{});
        else if (c == 1) gather(std::integral_constant<int, 1>{});
        else gather(std::integral_constant<int, 2>{});
    }
    __syncthreads();
    if (in_a) {
        DftP2<Q, true>::run(u);
        double2* dst = Y + n2 * P + p;
#pragma unroll
        for (int kb = 0; kb < Q; ++kb) {
            const int kq = 3 * kb + c;
            dst[kq * NB * P] = cmulc2(u[kb], ldtwn(tw, n2 * kq));
        }
    }
    __syncthreads();
    if (in_b) {
        const double2* src = Y + (k1 * NB) * P + p;
        double2 v[H];
        if (h == 0) {
#pragma unroll
            for (int m = 0; m < H; ++m) v[m] = cadd2(src[m * P], src[(m + H) * P]);
        } else {
#pragma unroll
            for (int m = 0; m < H; ++m) v[m] = csub2(src[m * P], src[(m + H) * P]);
            twiddle_odd_half<true>(v, std::make_integer_sequence<int, H>{});
        }
        DftP2<H, true>::run(v);
        // v[m] = (v1, v2)[j], j = k1 + NA (2 m + h): scatter to grid positions of the two lines
        double* o1 = X + (2 * p) * LX;
        double* o2 = o1 + LX;
#pragma unroll
        for (int m = 0; m < H; ++m) {
            const int j = k1 + NA * (2 * m + h);
            const int pos = (2 * j < N) ? 2 * j : 2 * (N - 1 - j) + 1;
            o1[pos] = v[m].x; o2[pos] = v[m].y;
        }
    }
    __syncthreads();
    // ---- store the grid lines (contiguous block)
    {
        const int cpl = N / 2, lane = tid & 31, nw = nthreads >> 5;
        for (int l = tid >> 5; l < nl; l += nw) {
            const double* src = X + l * LX;
            double* dst = a.out + (l0 + l) * N;
            for (int ch = lane; ch < cpl; ch += 32)
                *reinterpret_cast<double2*>(dst + 2 * ch) = *reinterpret_cast<const double2*>(src + 2 * ch);
        }
    }
}

template <int Q, int NB, int P>
__global__ void __launch_bounds__((ChGeom<Q, NB, P>::THREADS), (ChGeom<Q, NB, P>::MINB))
k_chfwd_regs(ChebArgs a)
{
    using G = ChGeom<Q, NB, P>;
    constexpr int NA = G::NA, N = G::N, H = NB / 2, LX = N + 2, CH_LINES = G::LINES;
    DB_SMEM(double, X);                                      // [16][LX] doubles, then Y = [N][P] double2
    double2* Y = reinterpret_cast<double2*>(X + CH_LINES * LX);
    const int tid = threadIdx.x, nthreads = blockDim.x;
    const int M = a.M;
    const int64_t l0 = (int64_t)blockIdx.x * CH_LINES;
    const int nl = (a.lines - l0 < CH_LINES) ? (int)(a.lines - l0) : CH_LINES;
    {
        const int cpl = N / 2, lane = tid & 31, nw = nthreads >> 5;
        for (int l = tid >> 5; l < CH_LINES; l += nw) {
            double* dst = X + l * LX;
            if (l < nl) {
                const double* src = a.in + (l0 + l) * N;
                for (int ch = lane; ch < cpl; ch += 32) db_cp_async16(dst + 2 * ch, src + 2 * ch);
            } else {
                for (int ch = lane; ch < cpl; ch += 32) { dst[2 * ch] = 0.0; dst[2 * ch + 1] = 0.0; }
            }
        }
        db_cp_commit();
        db_cp_wait<0>();
    }
    __syncthreads();
    const int p = tid & (P - 1), r = tid >> G::LOGP;
    const bool in_1 = r < 2 * NA, in_2 = r < 3 * NB;
    const int j1 = r % NA, h = r / NA;
    const int k2 = r % NB, c = r / NB;
    const double* __restrict__ tw = a.twn;
    if (in_1) {
        // stage 1: v[j] = (g1, g2)[pos(j)], j = j1 + NA j2; size-NB DFT over j2, outputs k2 = 2 m + h
        const double* g1 = X + (2 * p) * LX;
        const double* g2 = g1 + LX;
        auto val = [&](int j2) -> double2 {
            const int j = j1 + NA * j2;
            const int pos = (2 * j < N) ? 2 * j : 2 * (N - 1 - j) + 1;
            return make_double2(g1[pos], g2[pos]);
        };
        double2 v[H];
        if (h == 0) {
#pragma unroll
            for (int m = 0; m < H; ++m) v[m] = cadd2(val(m), val(m + H));
        } else {
#pragma unroll
            for (int m = 0; m < H; ++m) v[m] = csub2(val(m), val(m + H));
            twiddle_odd_half<false>(v, std::make_integer_sequence<int, H>{});
        }
        DftP2<H, false>::run(v);
        double2* dst = Y + (j1 * NB + h) * P + p;
#pragma unroll
        for (int m = 0; m < H; ++m) {
            const int kq = 2 * m + h;
            dst[(2 * m) * P] = (kq == 0) ? v[m] : cmul2(v[m], ldtwn(tw, j1 * kq));
        }
    }
    __syncthreads();
    double2 z[Q];
    if (in_2) {
        const double2* src = Y + k2 * P + p;
        if (c == 0) residue_gather<0, Q>(z, src, NB * P);
        else if (c == 1) residue_gather<1, Q>(z, src, NB * P);
        else residue_gather<2, Q>(z, src, NB * P);
        DftP2<Q, false>::run(z);
    }
    __syncthreads();
    if (in_2) {
        // full spectrum in natural order: Y[k][p] = Z_k, k = NB k1 + k2, k1 = c + 3 kb
        double2* dst = Y + (k2 * P) + p;
#pragma unroll
        for (int kb = 0; kb < Q; ++kb) dst[(NB * (3 * kb + c)) * P] = z[kb];
    }
    __syncthreads();
    // ---- coefficients of both lines of every pair into X[line][k] (k < Kin), scaled, odd modes negated
    const int Kin = M < N ? M : N;
    {
        const double s0 = 0.5 / N * 1.7724538509055160272981674833411;      // sqrt(pi)/(2N)
        const double s1 = 1.0 / N * 1.2533141373155002512078826424055;      // sqrt(pi/2)/N
        const int lane = tid & 31, w = tid >> 5, nw = nthreads >> 5;
        constexpr int PL = P < 4 ? P : 4, KL = 32 / PL, PH = P / PL;
        const int kk = lane / PL;
        for (int wt = w; wt < PH * ((Kin + KL - 1) / KL); wt += nw) {
            const int k = (wt / PH) * KL + kk, pp = (lane % PL) + PL * (wt % PH);
            if (k >= Kin) continue;
            double* x1 = X + (2 * pp) * LX;
            double* x2 = x1 + LX;
            const double2 za = Y[k * P + pp];
            const double2 zb = Y[((k == 0) ? 0 : N - k) * P + pp];
            const double2 S = make_double2(za.x + zb.x, za.y - zb.y);            // Z_k + conj Z_{n-k}
            const double2 D = make_double2(za.y + zb.y, zb.x - za.x);            // (Z_k - conj Z_{n-k}) / i
            const double2 q = ldtwn(a.twq, k);
            const double sc = ((k == 0) ? s0 : s1) * ((k & 1) ? -1.0 : 1.0);
            x1[k] = sc * (q.x * S.x - q.y * S.y);
            x2[k] = sc * (q.x * D.x - q.y * D.y);
        }
    }
    __syncthreads();
    // ---- store with the banded conversion applied: out[i] = sum_d diag[d][i] cof[i + d]
    {
        // one warp per line at a time, two adjacent outputs per lane (16-byte stores).  All diagonal values of an output pair
        // are loaded BEFORE the multiply-adds (not one dependent global load of diag[d][i] in front of every FMA with a
        // runtime trip count, which stalls the warp on every term)
        constexpr int MAXD = 8;
        const int nd = a.nd, lane = tid & 31, nw = nthreads >> 5;
        const double* __restrict__ dg = a.diags;
        for (int l = tid >> 5; l < nl; l += nw) {
            const double* cf = X + l * LX;
            double* dst = a.out + (l0 + l) * M;
            for (int i = 2 * lane; i < M; i += 64) {
                double acc0 = 0.0, acc1 = 0.0;
                if (nd == 0) {
                    acc0 = (i < Kin) ? cf[i] : 0.0; acc1 = (i + 1 < Kin) ? cf[i + 1] : 0.0;
                } else if (nd <= MAXD) {
                    double2 dv[MAXD];
                    double cv[MAXD + 1];
#pragma unroll
                    for (int d = 0; d < MAXD; ++d)
                        dv[d] = (d < nd) ? __ldg(reinterpret_cast<const double2*>(dg + (int64_t)d * M + i)) : make_double2(0.0, 0.0);
#pragma unroll
                    for (int d = 0; d <= MAXD; ++d) cv[d] = (d <= nd && i + d < Kin) ? cf[i + d] : 0.0;
#pragma unroll
                    for (int d = 0; d < MAXD; ++d) { acc0 = fma(dv[d].x, cv[d], acc0); acc1 = fma(dv[d].y, cv[d + 1], acc1); }
                } else {
                    for (int d = 0; d < nd; ++d) {
                        if (i + d < Kin) acc0 = fma(dg[(int64_t)d * M + i], cf[i + d], acc0);
                        if (i + 1 + d < Kin) acc1 = fma(dg[(int64_t)d * M + i + 1], cf[i + 1 + d], acc1);
                    }
                }
                *reinterpret_cast<double2*>(dst + i) = make_double2(acc0, acc1);
            }
        }
    }
}

template <int Q, int NB>
int launch_cheb(bool fwd, const ChebArgs& a, void* stream)
{
    // small transforms keep the tall tile (their CTAs are small anyway)
    constexpr int P = 3 * Q * NB < 192 ? 8 : 4;
    using G = ChGeom<Q, NB, P>;
    const int64_t blocks = (a.lines + G::LINES - 1) / G::LINES;
#ifndef DB_EMU
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(k_chbwd_regs<Q, NB, P>, cudaFuncAttributeMaxDynamicSharedMemorySize, DB_MAX_SMEM);
        cudaFuncSetAttribute(k_chfwd_regs<Q, NB, P>, cudaFuncAttributeMaxDynamicSharedMemorySize, DB_MAX_SMEM);
        cudaFuncSetAttribute(k_chbwd_regs<Q, NB, P>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
        cudaFuncSetAttribute(k_chfwd_regs<Q, NB, P>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
        attr = true;
    }
#endif
    if (fwd) DB_LAUNCH((k_chfwd_regs<Q, NB, P>), dim3((unsigned)blocks), dim3(G::THREADS), G::SMEM, stream, a);
    else DB_LAUNCH((k_chbwd_regs<Q, NB, P>), dim3((unsigned)blocks), dim3(G::THREADS), G::SMEM, stream, a);
    return db_check_launch(fwd ? "cheb_forward(regs)" : "cheb_backward(regs)");
}

static int regs_num_sms()
{
#ifdef DB_EMU
    return 1;                    // tests: several tiles per persistent CTA
#else
    return db_num_sms();
#endif
}

// CTAs of `kern` resident on one SM: the persistent grids launch exactly this many per SM (more would run as a second wave)
template <class K> int resident_per_sm(K kern, int threads, size_t bytes, int fit)
{
#ifdef DB_EMU
    (void)kern; (void)threads; (void)bytes;
    return fit;
#else
    int nb = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, threads, bytes) != cudaSuccess || nb < 1) return fit;
    return nb;
#endif
}

template <int Q, int NB>
size_t regs_smem() { return (size_t)2 * 3 * Q * NB * RR_P * sizeof(double2); }

template <int Q, int NB>
void regs_attrs()
{
    constexpr int P = RR_P;
#ifndef DB_EMU
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(k_rbwd_regs<Q, NB, P, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, DB_MAX_SMEM);
        cudaFuncSetAttribute(k_rbwd_regs<Q, NB, P, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, DB_MAX_SMEM);
        cudaFuncSetAttribute(k_rfwd_regs<Q, NB, P>, cudaFuncAttributeMaxDynamicSharedMemorySize, DB_MAX_SMEM);
        cudaFuncSetAttribute(k_rbwd_regs<Q, NB, P, false>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
        cudaFuncSetAttribute(k_rbwd_regs<Q, NB, P, true>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
        cudaFuncSetAttribute(k_rfwd_regs<Q, NB, P>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
        attr = true;
    }
#endif
}

template <int Q, int NB>
int launch_regs(bool fwd, const RegArgs& a, int64_t outer, void* stream)
{
    constexpr int P = RR_P, THREADS = RegGeom<Q, NB, P>::THREADS;
    const size_t bytes = regs_smem<Q, NB>();
    TileWalk w;
    w.tiles_per_outer = a.inner / (2 * P);
    w.total = w.tiles_per_outer * outer;
    // persistent grid: as many CTAs as are resident (at n = 384, P = 8: 2 per SM of 96 KB each for the plain backward, 1 for
    // the forward and derivative backward, which take the whole register file), never more than there are tiles
    int per_sm = (int)((size_t)(226 * 1024) / (bytes + 1024));
    if (per_sm < 1) per_sm = 1;
    if (per_sm > 8) per_sm = 8;
    regs_attrs<Q, NB>();
    if (fwd) per_sm = resident_per_sm(k_rfwd_regs<Q, NB, P>, THREADS, bytes, per_sm);
    else if (a.deriv > 0) per_sm = resident_per_sm(k_rbwd_regs<Q, NB, P, true>, THREADS, bytes, per_sm);
    else per_sm = resident_per_sm(k_rbwd_regs<Q, NB, P, false>, THREADS, bytes, per_sm);
    int64_t nblk = (int64_t)regs_num_sms() * per_sm;
    if (nblk > w.total) nblk = w.total;
    dim3 grid((unsigned)nblk);
    if (fwd) DB_LAUNCH((k_rfwd_regs<Q, NB, P>), grid, dim3(THREADS), bytes, stream, a, w);
    else if (a.deriv > 0) DB_LAUNCH((k_rbwd_regs<Q, NB, P, true>), grid, dim3(THREADS), bytes, stream, a, w);
    else DB_LAUNCH((k_rbwd_regs<Q, NB, P, false>), grid, dim3(THREADS), bytes, stream, a, w);
    return db_check_launch(fwd ? "rfft_forward(regs)" : "rfft_backward(regs)");
}

// CTAs per SM of the fused x pass (its persistent grid is this times the SM count)
template <int Q, int NB>
int x_products_per_sm(size_t bytes)
{
    constexpr int P = RR_P;
    using X = XpGeom<Q, NB, P>;
    int fit = (int)((size_t)(226 * 1024) / (bytes + 1024));
    if (fit > X::MINB) fit = X::MINB;
    if (fit < 1) fit = 1;
#ifndef DB_EMU
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(k_rfft_x_products<Q, NB, P>, cudaFuncAttributeMaxDynamicSharedMemorySize, DB_MAX_SMEM);
        cudaFuncSetAttribute(k_rfft_x_products<Q, NB, P>, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
        attr = true;
    }
#endif
    return resident_per_sm(k_rfft_x_products<Q, NB, P>, X::THREADS, bytes, fit);
}

template <int Q, int NB>
int launch_x_products(const XProdArgs& a, int32_t n_held, void* stream)
{
    constexpr int P = RR_P;
    using X = XpGeom<Q, NB, P>;
    const size_t bytes = X::smem(a.M, n_held);
    if (bytes > (size_t)DB_MAX_SMEM) {
        db_set_error("rfft_x_products: %d held factors at n = %d need %zu bytes of shared memory", (int)n_held, X::N, bytes);
        return 1;
    }
    const int64_t total = a.inner / (2 * P);
    int64_t nblk = (int64_t)regs_num_sms() * x_products_per_sm<Q, NB>(bytes);
    if (nblk > total) nblk = total;
    DB_LAUNCH((k_rfft_x_products<Q, NB, P>), dim3((unsigned)nblk), dim3(X::THREADS), bytes, stream, a, total);
    return db_check_launch("rfft_x_products");
}

template <int Q, int NB>
int blocks_per_sm(int kind, int32_t n_coeff, int32_t n_held)
{
    constexpr int P = RR_P;
    if (kind < 0 || kind > 2) return -1;
    if (kind == 2) return x_products_per_sm<Q, NB>(XpGeom<Q, NB, P>::smem(n_coeff, n_held));
    regs_attrs<Q, NB>();
    const size_t bytes = regs_smem<Q, NB>();
    int fit = (int)((size_t)(226 * 1024) / (bytes + 1024));
    fit = fit < 1 ? 1 : (fit > 8 ? 8 : fit);
    if (kind == 1) return resident_per_sm(k_rfwd_regs<Q, NB, P>, RegGeom<Q, NB, P>::THREADS, bytes, fit);
    return resident_per_sm(k_rbwd_regs<Q, NB, P, false>, RegGeom<Q, NB, P>::THREADS, bytes, fit);
}

static long long g_regs_launches = 0;
}  // namespace

extern "C" long long db_rfft_regs_launches(void) { return g_regs_launches; }

// Returns -1 if the register kernels do not cover this case (the caller falls back to the generic shared-memory
// kernel), otherwise the launch status.
int db_rfft_regs_try(bool fwd, const db_fft_plan* plan, const double* in, double* out, int64_t outer, int32_t n_coeff,
                     int64_t inner, int32_t deriv, double kscale, void* stream,
                     int32_t in_rpb, int64_t in_blk_stride, int32_t out_rpb, int64_t out_blk_stride,
                     int32_t out_peers, double* const* out_blk_ptr)
{
    const int n = plan->n;
    if (!plan->half || plan->twn == nullptr) return -1;
    if (inner < RR_LINES || inner % RR_LINES != 0 || deriv > 4) return -1;
    if (n_coeff % 2 != 0 || n_coeff < 2 || (int64_t)3 * n_coeff > (int64_t)2 * n) return -1;
    if ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) return -1;
    RegArgs a;
    a.in = in; a.out = out; a.twn = plan->twn; a.inner = inner; a.M = n_coeff; a.deriv = deriv; a.kscale = kscale;
    a.in_rpb = in_rpb; a.in_blk_stride = in_blk_stride; a.out_rpb = out_rpb; a.out_blk_stride = out_blk_stride;
    a.out_peers = 0;
    for (int i = 0; i < 8; ++i) a.out_blk_ptr[i] = nullptr;
    if (out_peers > 0) {
        if (out_peers > 8 || out_rpb <= 0 || out_blk_ptr == nullptr) return -1;
        a.out_peers = out_peers;
        for (int i = 0; i < out_peers; ++i) {
            if (reinterpret_cast<uintptr_t>(out_blk_ptr[i]) & 15) return -1;
            a.out_blk_ptr[i] = out_blk_ptr[i];
        }
    }
    if (((in_rpb ? in_blk_stride : 0) | (out_rpb ? out_blk_stride : 0)) & 1) return -1;          // 16-byte alignment of every block
    ++g_regs_launches;
    switch (n) {
        case 384: return launch_regs<8, 16>(fwd, a, outer, stream);
        case 192: return launch_regs<4, 16>(fwd, a, outer, stream);
        case 96:  return launch_regs<4, 8>(fwd, a, outer, stream);
        case 48:  return launch_regs<2, 8>(fwd, a, outer, stream);
        case 24:  return launch_regs<2, 4>(fwd, a, outer, stream);
        case 768: return launch_regs<8, 32>(fwd, a, outer, stream);
        default: --g_regs_launches; return -1;
    }
}

// Chebyshev on contiguous lines (inner == 1): returns -1 if not covered (generic kernel in fft.cu takes over).
// backward: plain DCT-III, optionally preceded (in shared memory) by the derivative pre-apply + the back-substitution
// of a conversion with only the main and the second super-diagonal (`sol2`, compact storage as db_band_lines stride 2);
// forward: conversion diagonals fused into the store.
int db_cheb_regs_try(bool fwd, const db_fft_plan* plan, const double* in, double* out, int64_t lines, int32_t n_coeff,
                     const double* diags, int32_t nd, const double* pre, int32_t npre, const double* sol2, void* stream)
{
    const int n = plan->n;
    if (plan->twn == nullptr || plan->twq == nullptr) return -1;
    if (n_coeff % 2 != 0 || n_coeff < 2 || n_coeff > n || lines > 2147483647LL * 4) return -1;
    if ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) return -1;
    ChebArgs a;
    a.in = in; a.out = out; a.twn = plan->twn; a.twq = plan->twq; a.diags = diags; a.lines = lines; a.M = n_coeff; a.nd = nd;
    a.pre = pre; a.npre = npre; a.sol2 = sol2;
    if (npre > 3 || (npre > 0 && sol2 == nullptr)) return -1;
    ++g_regs_launches;
    switch (n) {
        case 384: return launch_cheb<8, 16>(fwd, a, stream);
        case 192: return launch_cheb<4, 16>(fwd, a, stream);
        case 96:  return launch_cheb<4, 8>(fwd, a, stream);
        case 48:  return launch_cheb<2, 8>(fwd, a, stream);
        case 24:  return launch_cheb<2, 4>(fwd, a, stream);
        default: --g_regs_launches; return -1;
    }
}

// Fused x pass of a quadratic right-hand side (k_rfft_x_products); every case it does not cover is an error: the caller checks
// coverage first (RealFourierTransform.x_products_supported mirrors these conditions).
extern "C" int db_rfft_x_products(const db_fft_plan* plan, const double* in, int64_t in_stride, double* out, int64_t out_stride,
                                  int32_t n_coeff, int64_t inner, double kscale, const db_xprod_item* items, int32_t n_items,
                                  const int32_t* loads, int32_t n_loads, int32_t n_held, void* stream)
{
    const int n = plan->n;
    const bool ok = plan->half && plan->twn != nullptr && inner >= RR_LINES && inner % RR_LINES == 0 && n_coeff % 2 == 0 &&
                    n_coeff >= 2 && (int64_t)3 * n_coeff <= (int64_t)2 * n && n_held >= 0 && n_held <= 3 && n_items > 0 &&
                    n_loads > 0 && in_stride % 2 == 0 && out_stride % 2 == 0 &&
                    ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
    if (!ok) {
        db_set_error("rfft_x_products: case not covered (n = %d, M = %d, inner = %lld, %d held factors)", n, (int)n_coeff,
                     (long long)inner, (int)n_held);
        return 1;
    }
    XProdArgs a;
    a.in = in; a.out = out; a.twn = plan->twn; a.inner = inner; a.in_stride = in_stride; a.out_stride = out_stride;
    a.M = n_coeff; a.kscale = kscale; a.items = items; a.n_items = n_items; a.loads = loads; a.n_loads = n_loads;
    ++g_regs_launches;
    switch (n) {
        case 384: return launch_x_products<8, 16>(a, n_held, stream);
        case 192: return launch_x_products<4, 16>(a, n_held, stream);
        case 96:  return launch_x_products<4, 8>(a, n_held, stream);
        case 48:  return launch_x_products<2, 8>(a, n_held, stream);
        case 24:  return launch_x_products<2, 4>(a, n_held, stream);
        default:
            --g_regs_launches;
            db_set_error("rfft_x_products: no kernel for n = %d", n);
            return 1;
    }
}

// Resident CTAs per SM of a register transform (kind 0: backward, 1: forward) or of the fused x pass (kind 2, with n_coeff rows
// and n_held held factors) at n grid points; -1 where no such kernel exists.
extern "C" int db_rfft_blocks_per_sm(int32_t kind, int32_t n, int32_t n_coeff, int32_t n_held)
{
    switch (n) {
        case 384: return blocks_per_sm<8, 16>(kind, n_coeff, n_held);
        case 192: return blocks_per_sm<4, 16>(kind, n_coeff, n_held);
        case 96:  return blocks_per_sm<4, 8>(kind, n_coeff, n_held);
        case 48:  return blocks_per_sm<2, 8>(kind, n_coeff, n_held);
        case 24:  return blocks_per_sm<2, 4>(kind, n_coeff, n_held);
        default: return -1;
    }
}
