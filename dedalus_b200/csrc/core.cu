// Error plumbing, version / device probes and small utility kernels.
#include "db_common.cuh"
#include <cstdarg>

static char g_last_error[512] = "";

void db_set_error(const char* fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
    va_end(ap);
}

int db_check_launch(const char* what)
{
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) {
        db_set_error("%s: kernel launch failed: %s", what, cudaGetErrorString(err));
        return 2;
    }
    return 0;
}

extern "C" const char* db_last_error(void) { return g_last_error; }
extern "C" int db_version(void) { return 100; }

int db_num_sms()
{
#ifdef DB_EMU
    return 132;                  // the emulation sizes grids as for an H100
#else
    static int n = 0;
    if (n == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    }
    return n;
#endif
}

extern "C" int db_device_arch(void)
{
#ifdef DB_EMU
    return 0;
#else
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { db_set_error("no CUDA device"); return -1; }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) { db_set_error("cudaGetDeviceProperties failed"); return -1; }
    return prop.major * 10 + prop.minor;
#endif
}

// |x| max reduction: per-block partial maxima combined with atomicMax on the ordered-int representation.  A NaN in the input
// propagates to the result, as np.max does: it wins every comparison on the way, and is published as the positive quiet NaN,
// whose bit pattern lies above every finite value and +inf.
__device__ __forceinline__ void db_publish_max(unsigned long long* out, double v)
{
    // non-negative doubles order like their bit patterns
    unsigned long long bits;
    memcpy(&bits, &v, sizeof(bits));
    if (v != v) bits = 0x7ff8000000000000ull;
#ifdef DB_EMU
    if (bits > *out) *out = bits;
#else
    atomicMax(out, bits);
#endif
}

__global__ void k_absmax(const double* __restrict__ x, int64_t count, unsigned long long* __restrict__ out)
{
    DB_SMEM(double, red);
    double m = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) {
        double v = fabs(x[i]);
        m = (v > m || v != v) ? v : m;           // a NaN wins and stays
    }
    red[threadIdx.x] = m;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) { double o = red[threadIdx.x + s]; if (o > red[threadIdx.x] || o != o) red[threadIdx.x] = o; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        // non-negative doubles order like their bit patterns
        db_publish_max(out, red[0]);
    }
}

extern "C" int db_absmax(const double* x, int64_t count, double* out, void* stream)
{
    // `out` must be zero-initialised by the caller (0.0 has an all-zero bit pattern)
    if (count <= 0) return 0;
    int64_t blocks = (count + 255) / 256;
    if (blocks > (int64_t)db_num_sms() * 8) blocks = (int64_t)db_num_sms() * 8;
    DB_LAUNCH(k_absmax, dim3((unsigned)blocks), dim3(256), 256 * sizeof(double), stream, x, count, reinterpret_cast<unsigned long long*>(out));
    return db_check_launch("absmax");
}


// advective CFL frequency maximum
struct CflArgs { const double* u[3]; const double* idx[3]; int ncomp; int64_t g0, g1, g2; };

__global__ void k_cfl_max(CflArgs a, unsigned long long* __restrict__ out)
{
    DB_SMEM(double, red);
    const int64_t total = a.g0 * a.g1 * a.g2;
    double m = 0.0;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i2 = e % a.g2; const int64_t q = e / a.g2;
        const int64_t i1 = q % a.g1; const int64_t i0 = q / a.g1;
        const int64_t ix[3] = {i0, i1, i2};
        double f = 0.0;
        for (int c = 0; c < a.ncomp; ++c) f += fabs(a.u[c][e]) * a.idx[c][ix[3 - a.ncomp + c]];
        m = (f > m || f != f) ? f : m;
    }
    red[threadIdx.x] = m;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) { double o = red[threadIdx.x + s]; if (o > red[threadIdx.x] || o != o) red[threadIdx.x] = o; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        db_publish_max(out, red[0]);
    }
}

extern "C" int db_cfl_max(const double* const* u, const double* const* inv_dx, int32_t ncomp, int64_t g0, int64_t g1, int64_t g2,
                          double* out, void* stream)
{
    if (ncomp < 1 || ncomp > 3) { db_set_error("cfl_max: ncomp must be 1..3"); return 1; }
    CflArgs a;
    for (int c = 0; c < 3; ++c) { a.u[c] = (c < ncomp) ? u[c] : nullptr; a.idx[c] = (c < ncomp) ? inv_dx[c] : nullptr; }
    a.ncomp = ncomp; a.g0 = g0; a.g1 = g1; a.g2 = g2;
    const int64_t total = g0 * g1 * g2;
    if (total <= 0) return 0;
    int64_t blocks = (total + 255) / 256;
    if (blocks > (int64_t)db_num_sms() * 8) blocks = (int64_t)db_num_sms() * 8;
    DB_LAUNCH(k_cfl_max, dim3((unsigned)blocks), dim3(256), 256 * sizeof(double), stream, a, reinterpret_cast<unsigned long long*>(out));
    return db_check_launch("cfl_max");
}

// advective CFL frequency maximum on spheres and spherical shells: sqrt(u_phi^2 + u_theta^2) * inv_h[ir] + |u_r| * inv_dr[ir]
// (S2AdvectiveCFL / Spherical3DAdvectiveCFL.compute_cfl_frequency, core/basis.py:6175-6212); arrays (n_ang, n_r), u_r may be NULL
__global__ void k_cfl_max_spherical(const double* __restrict__ up, const double* __restrict__ ut, const double* __restrict__ ur,
                                    const double* __restrict__ inv_h, const double* __restrict__ inv_dr, int64_t n_ang, int64_t n_r,
                                    unsigned long long* __restrict__ out)
{
    DB_SMEM(double, red);
    const int64_t total = n_ang * n_r;
    double m = 0.0;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t ir = e % n_r;
        double f = sqrt(up[e] * up[e] + ut[e] * ut[e]) * inv_h[ir];
        if (ur) f += fabs(ur[e]) * inv_dr[ir];
        m = (f > m || f != f) ? f : m;
    }
    red[threadIdx.x] = m;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) { double o = red[threadIdx.x + s]; if (o > red[threadIdx.x] || o != o) red[threadIdx.x] = o; }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        db_publish_max(out, red[0]);
    }
}

extern "C" int db_cfl_max_spherical(const double* u_phi, const double* u_theta, const double* u_r, const double* inv_h, const double* inv_dr,
                                    int64_t n_ang, int64_t n_r, double* out, void* stream)
{
    const int64_t total = n_ang * n_r;
    if (total <= 0) return 0;
    int64_t blocks = (total + 255) / 256;
    if (blocks > (int64_t)db_num_sms() * 8) blocks = (int64_t)db_num_sms() * 8;
    DB_LAUNCH(k_cfl_max_spherical, dim3((unsigned)blocks), dim3(256), 256 * sizeof(double), stream, u_phi, u_theta, u_r, inv_h, inv_dr,
              n_ang, n_r, reinterpret_cast<unsigned long long*>(out));
    return db_check_launch("cfl_max_spherical");
}
