// Boltzmann-machine learning of a Potts model (evc_code_counts, evc_bm_update; contracts in include/evcplm.h).
//
// evc_code_counts: exact one- and two-site counts of N code rows in the layout of x.  A "unit" is a site (q
// counters, [i q + a]) or a site pair i < j (q q counters, [pair][a][b]); units are numbered sites first, then pairs
// in row-major order, so unit u's counters start at its offset in x.  One CTA owns a contiguous range of units of
// one kind, keeps their histograms in shared memory and walks all N rows in stages of COUNT_STAGE_BYTES of codes:
// consecutive threads take consecutive units of the same row, so a warp's shared-memory increments never collide.
// At the end the CTA stores its histograms with plain stores: every counter is written exactly once, there is no
// memset and no global atomic, and the result does not depend on the launch.
//
// evc_bm_update: one grid-stride pass over x: read theta, the count and the target, write theta, and fold
// |c/M - f| into a per-region maximum (a warp max, then atomicMax on the bit pattern, which orders like the value
// for non-negative doubles).
#include "../../include/evcplm.h"

#include <math.h>

#include <algorithm>
#include <string>

#include "common.cuh"

namespace evc {

constexpr int COUNT_THREADS = 512;
constexpr int COUNT_HIST_BYTES = 64 * 1024;     // histograms of one CTA
constexpr int COUNT_STAGE_BYTES = 32 * 1024;    // staged code rows of one CTA
constexpr int COUNT_MAX_L = COUNT_STAGE_BYTES;  // one whole row must fit the stage
constexpr int UPDATE_THREADS = 256;

struct CountPlan {
    int units_per_site_cta, units_per_pair_cta;
    int64_t site_ctas, pair_ctas;
    int rows_per_stage;
};

static CountPlan count_plan(int L, int q)
{
    CountPlan p;
    const int64_t npairs = (int64_t)L * (L - 1) / 2;
    p.units_per_site_cta = std::min<int64_t>(L, COUNT_HIST_BYTES / (4 * q));
    p.units_per_pair_cta = (int)std::min<int64_t>(std::max<int64_t>(npairs, 1), COUNT_HIST_BYTES / (4 * q * q));
    p.site_ctas = ceil_div(L, p.units_per_site_cta);
    p.pair_ctas = npairs ? ceil_div(npairs, p.units_per_pair_cta) : 0;
    p.rows_per_stage = std::max(1, COUNT_STAGE_BYTES / L);
    return p;
}

// blocks [0, site_ctas) count sites, the rest count pairs; smem = [histograms (uint32)][unit sites (2 x int32)][codes]
__global__ void __launch_bounds__(COUNT_THREADS)
code_counts_kernel(const uint8_t *__restrict__ codes, int64_t N, int L, int q, int units_per_site_cta,
                   int units_per_pair_cta, int site_ctas, int rows_per_stage, uint32_t *__restrict__ counts)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const bool pairs = (int)blockIdx.x >= site_ctas;
    const int64_t npairs = (int64_t)L * (L - 1) / 2;
    const int per = pairs ? units_per_pair_cta : units_per_site_cta;
    const int width = pairs ? q * q : q;
    const int64_t u0 = pairs ? (int64_t)(blockIdx.x - site_ctas) * per : (int64_t)blockIdx.x * per;
    const int units = (int)min((int64_t)per, (pairs ? npairs : L) - u0);
    uint32_t *hist = reinterpret_cast<uint32_t *>(smem_raw);
    int *ui = reinterpret_cast<int *>(hist + (size_t)per * width);
    int *uj = ui + per;
    uint8_t *stage = reinterpret_cast<uint8_t *>(uj + per);
    for (int e = threadIdx.x; e < units * width; e += blockDim.x) hist[e] = 0;
    for (int k = threadIdx.x; k < units; k += blockDim.x) {
        const int64_t u = u0 + k;
        if (pairs) {        // pair u = i L - i (i + 1) / 2 + (j - i - 1): find i by walking the rows of the triangle
            int i = 0;
            int64_t first = 0;
            while (first + (L - 1 - i) <= u) { first += L - 1 - i; i++; }
            ui[k] = i;
            uj[k] = i + 1 + (int)(u - first);
        } else {
            ui[k] = (int)u;
            uj[k] = (int)u;
        }
    }
    const int mi = pairs ? q : 1, mj = pairs ? 1 : 0;
    for (int64_t n0 = 0; n0 < N; n0 += rows_per_stage) {
        const int rows = (int)min((int64_t)rows_per_stage, N - n0);
        __syncthreads();                        // the previous stage is consumed (and the unit table is written)
        const uint8_t *src = codes + n0 * L;
        for (int e = threadIdx.x; e < rows * L; e += blockDim.x) stage[e] = src[e];
        __syncthreads();
        for (int e = threadIdx.x; e < rows * units; e += blockDim.x) {
            const int r = e / units, k = e - r * units;
            const uint8_t *row = stage + (size_t)r * L;
            atomicAdd(&hist[k * width + row[ui[k]] * mi + row[uj[k]] * mj], 1u);
        }
    }
    __syncthreads();
    uint32_t *out = counts + (pairs ? (int64_t)L * q + u0 * width : u0 * width);
    for (int e = threadIdx.x; e < units * width; e += blockDim.x) out[e] = hist[e];
}

__device__ __forceinline__ void max_to(double v, unsigned long long *dst)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    if ((threadIdx.x & 31) == 0 && v > 0.0) atomicMax(dst, (unsigned long long)__double_as_longlong(v));
}

// g = (c/M - f) + lam2 theta; theta <- fp32_rn(theta - eta g); every operation rounded on its own (no FMA)
__global__ void __launch_bounds__(UPDATE_THREADS)
bm_update_kernel(float *__restrict__ x, const uint32_t *__restrict__ counts, double M, const float *__restrict__ f,
                 int64_t n, int64_t Lq, double eta, double lam2_h, double lam2_J, unsigned long long *__restrict__ stats)
{
    double dev_h = 0.0, dev_J = 0.0;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
        const double th = (double)x[k];
        const double d = __dsub_rn(__ddiv_rn((double)counts[k], M), (double)f[k]);
        const double g = __dadd_rn(d, __dmul_rn(k < Lq ? lam2_h : lam2_J, th));
        x[k] = __double2float_rn(__dsub_rn(th, __dmul_rn(eta, g)));
        if (k < Lq) dev_h = fmax(dev_h, fabs(d));
        else dev_J = fmax(dev_J, fabs(d));
    }
    max_to(dev_h, stats);
    max_to(dev_J, stats + 1);
}

}  // namespace evc

using namespace evc;

extern "C" {

int evc_code_counts(const uint8_t *d_codes, int64_t N, int32_t L, int32_t q, uint32_t *d_counts, void *stream)
{
    const std::string name = "evc_code_counts";
    if (!d_codes || !d_counts) { set_error(name + ": null pointer"); return 1; }
    if (q < 2 || q > 32) {
        set_error(name + ": unsupported number of states q=" + std::to_string(q) + " (2 <= q <= 32)");
        return 1;
    }
    if (L < 1 || L > COUNT_MAX_L) {
        set_error(name + ": L=" + std::to_string(L) + " out of range (1 <= L <= " + std::to_string(COUNT_MAX_L) + ")");
        return 1;
    }
    if (N < 1 || N > INT32_MAX) { set_error(name + ": N must be in [1, 2^31 - 1]"); return 1; }
    const CountPlan p = count_plan(L, q);
    const int per_max = std::max(p.units_per_site_cta, p.units_per_pair_cta);
    const int width_max = std::max(p.units_per_site_cta * q, p.units_per_pair_cta * q * q);
    const size_t smem = (size_t)width_max * 4 + (size_t)per_max * 8 + (size_t)p.rows_per_stage * L;
    EVC_CUDA(cudaFuncSetAttribute(code_counts_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    code_counts_kernel<<<(unsigned)(p.site_ctas + p.pair_ctas), COUNT_THREADS, smem,
                         reinterpret_cast<cudaStream_t>(stream)>>>(d_codes, N, L, q, p.units_per_site_cta,
                                                                   p.units_per_pair_cta, (int)p.site_ctas,
                                                                   p.rows_per_stage, d_counts);
    EVC_KERNEL_CHECK();
    return 0;
}

int evc_bm_update(float *d_x, const uint32_t *d_counts, int64_t M, const float *d_f, int64_t n, int32_t Lq,
                  double eta, double lam2_h, double lam2_J, double *d_stats, void *stream)
{
    const std::string name = "evc_bm_update";
    if (!d_x || !d_counts || !d_f || !d_stats) { set_error(name + ": null pointer"); return 1; }
    if (M < 1) { set_error(name + ": M must be >= 1"); return 1; }
    if (n < 1 || Lq < 0 || Lq > n) { set_error(name + ": need n >= 1 and 0 <= Lq <= n"); return 1; }
    if (!isfinite(eta) || !isfinite(lam2_h) || !isfinite(lam2_J)) {
        set_error(name + ": eta, lam2_h and lam2_J must be finite");
        return 1;
    }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    EVC_CUDA(cudaMemsetAsync(d_stats, 0, 2 * sizeof(double), st));
    const int64_t blocks = std::min<int64_t>(ceil_div(n, UPDATE_THREADS), 132 * 16);
    bm_update_kernel<<<(unsigned)blocks, UPDATE_THREADS, 0, st>>>(d_x, d_counts, (double)M, d_f, n, Lq, eta, lam2_h,
                                                                   lam2_J,
                                                                   reinterpret_cast<unsigned long long *>(d_stats));
    EVC_KERNEL_CHECK();
    return 0;
}

}  // extern "C"
