// a8: device-side vector algebra for L-BFGS (SURVEY.md 8a row a8) and the EC Frobenius norms (a10).
// plmc drives libLBFGS on the host CPU; here the n-vector work (n = L*q + L(L-1)/2*q^2, 8.8M floats
// at L=200) stays in HBM and every scalar (dot products, alpha/beta of the two-loop recursion) stays
// on the device in double, so a direction costs no host round trip.  These are the kernels of evc_plm_fit
// (fit.cu) and of the ABI entry points evc_vec_dot, evc_lbfgs_* and evc_plm_add_regulariser alike.
//
//   trial point      x_try = x + t d                                    (1 kernel, 3 vector passes)
//   regulariser      g += 2 lambda x fused with the five reductions lambda|x|^2, g.d, g.g, |h|^2, |J|^2
//   two-loop         2*bound+1 fused kernels "d += c v; partial(u.d)" (4 vector passes each) with the
//                    coefficients alpha/beta kept on the device
// Every reduction runs on one fixed grid (RED_BLOCKS CTAs) and sums their partials in one fixed tree, so the result
// does not depend on the GPU and every rank of a data-parallel run takes bit-identical decisions without
// broadcasting anything.
#include <algorithm>
#include <map>
#include <mutex>
#include <utility>

#include "common.cuh"
#include "internal.h"

namespace evc {

constexpr int RED_THREADS = 256;
constexpr int RED_NRED = RED_PARTIALS / RED_BLOCKS;   // reductions of the regulariser kernel
constexpr int64_t FX_LIMB_BITS = 18;
constexpr double FX_SCALE = 65536.0;                  // fixed-point resolution 2^-16 of the packed -loglk

// Reduction partials of the ABI entry points are kept per (device, stream): two problems / threads / streams on one
// device do not share a buffer (ADVICE r1).  Buffers live for the lifetime of the process (47 KB each).
static std::mutex g_scratch_mutex;
static std::map<std::pair<int, cudaStream_t>, double *> g_scratch;

double *reduction_scratch(cudaStream_t st)
{
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) {
        set_error("reduction_scratch: bad device");
        return nullptr;
    }
    std::lock_guard<std::mutex> lock(g_scratch_mutex);
    double *&slot = g_scratch[std::make_pair(dev, st)];
    if (!slot && cudaMalloc(&slot, RED_PARTIALS * sizeof(double)) != cudaSuccess) {
        slot = nullptr;
        set_error("reduction_scratch: cudaMalloc failed");
        return nullptr;
    }
    return slot;
}

__device__ __forceinline__ double cta_sum(double v, double *s_red)
{
    v = warp_sum(v);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) s_red[warp] = v;
    __syncthreads();
    double tot = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) tot += s_red[w];
    return tot;   // valid on thread 0
}

// fixed-tree sum of RED_BLOCKS partials by one CTA of 1024 threads; result valid on thread 0
__device__ __forceinline__ double final_sum(const double *__restrict__ partial, double *s_red)
{
    const int tid = threadIdx.x;
    double v = 0.0;
    for (int e = tid; e < RED_BLOCKS; e += 1024) v += partial[e];
    __syncthreads();
    s_red[tid] = v;
    __syncthreads();
    for (int o = 512; o > 0; o >>= 1) {
        if (tid < o) s_red[tid] += s_red[tid + o];
        __syncthreads();
    }
    return s_red[0];
}

__global__ void step_kernel(float *__restrict__ xt, const float *__restrict__ x, const float *__restrict__ d, float t,
                            int64_t n)
{
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x)
        xt[e] = fmaf(t, d[e], x[e]);
}

int vec_step(float *xt, const float *x, const float *d, float t, int64_t n, cudaStream_t st)
{
    step_kernel<<<RED_BLOCKS, RED_THREADS, 0, st>>>(xt, x, d, t, n);
    EVC_KERNEL_CHECK();
    return 0;
}

// -loglk -> three fixed-point limbs (floats holding integers < 2^18) behind the gradient.  The 4th float is 0, or NaN
// when -loglk cannot be carried (NaN, +-inf, or beyond the clamp): a NaN survives every float sum, so one such rank
// makes the decoded -loglk NaN on all ranks, which is what a single rank reads from its own evaluation.
__global__ void pack_fx_kernel(const double *__restrict__ fx, float *__restrict__ limbs)
{
    const double raw = fx[0] * FX_SCALE;
    const double lim = 9.0e15;                      // |q| < 2^53: the top limb stays below 2^17 per rank (exact sums up to 64 ranks)
    const double v = fmin(fmax(raw, -lim), lim);    // fmax(NaN, -lim) is -lim
    const long long q = llrint(v);
    const long long mask = (1ll << FX_LIMB_BITS) - 1;
    limbs[0] = (float)(q & mask);
    limbs[1] = (float)((q >> FX_LIMB_BITS) & mask);
    limbs[2] = (float)(q >> (2 * FX_LIMB_BITS));    // arithmetic shift keeps the sign
    limbs[3] = v == raw ? 0.f : nanf("");
}

// the limbs (summed over the ranks) -> -loglk; NaN if any rank flagged its -loglk in the 4th float
__device__ __forceinline__ double unpack_fx(const float *__restrict__ limbs)
{
    if (limbs[3] != 0.f) return nan("");
    const long long q = (long long)limbs[0] + ((long long)limbs[1] << FX_LIMB_BITS) +
                        ((long long)limbs[2]) * (1ll << (2 * FX_LIMB_BITS));
    return (double)q / FX_SCALE;
}

__global__ void unpack_fx_kernel(const float *__restrict__ limbs, double *__restrict__ fx) { fx[0] = unpack_fx(limbs); }

int fx_pack(const double *fx, float *limbs, cudaStream_t st)
{
    pack_fx_kernel<<<1, 1, 0, st>>>(fx, limbs);
    EVC_KERNEL_CHECK();
    return 0;
}

int fx_unpack(const float *limbs, double *fx, cudaStream_t st)
{
    unpack_fx_kernel<<<1, 1, 0, st>>>(limbs, fx);
    EVC_KERNEL_CHECK();
    return 0;
}

// g += 2 lambda x; partials of {lambda |x|^2, g.d, g.g, |h|^2, |J|^2}   (d may be null)
__global__ void reg_dots_kernel(const float *__restrict__ x, float *__restrict__ g, const float *__restrict__ d,
                                int64_t n, int64_t nh, float lambda_h, float lambda_J, double *__restrict__ partial)
{
    __shared__ double s_red[32];
    double a_reg = 0.0, a_dg = 0.0, a_gg = 0.0, a_h = 0.0, a_J = 0.0;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        const bool is_h = e < nh;
        const float lam = is_h ? lambda_h : lambda_J;
        const float xv = x[e];
        const float gv = g[e] + 2.f * lam * xv;
        g[e] = gv;
        const double xx = (double)xv * (double)xv;
        a_reg += (double)lam * xx;
        if (is_h) a_h += xx; else a_J += xx;
        a_gg += (double)gv * (double)gv;
        if (d != nullptr) a_dg += (double)gv * (double)d[e];
    }
    double r[RED_NRED] = {a_reg, a_dg, a_gg, a_h, a_J};
#pragma unroll
    for (int k = 0; k < RED_NRED; k++) {
        const double tot = cta_sum(r[k], s_red);
        if (threadIdx.x == 0) partial[k * RED_BLOCKS + blockIdx.x] = tot;
    }
}

__global__ void __launch_bounds__(1024)
reg_final_kernel(const double *__restrict__ partial, const double *__restrict__ fx_data,
                 const float *__restrict__ limbs, double *__restrict__ nll_out, double *__restrict__ fx_out,
                 double *__restrict__ dots)
{
    __shared__ double s_red[1024];
    double out[RED_NRED];
    for (int k = 0; k < RED_NRED; k++) out[k] = final_sum(partial + k * RED_BLOCKS, s_red);
    if (threadIdx.x == 0) {
        const double nll = limbs != nullptr ? unpack_fx(limbs) : fx_data[0];
        if (nll_out != nullptr) nll_out[0] = nll;
        fx_out[0] = nll + out[0];
        if (dots != nullptr)
            for (int k = 1; k < RED_NRED; k++) dots[k - 1] = out[k];
    }
}

int regulariser(const float *x, float *g, const float *d, int64_t n, int64_t nh, float lambda_h, float lambda_J,
                const double *fx_data, const float *limbs, double *nll_out, double *fx_out, double *dots,
                double *partial, cudaStream_t st)
{
    reg_dots_kernel<<<RED_BLOCKS, RED_THREADS, 0, st>>>(x, g, d, n, nh, lambda_h, lambda_J, partial);
    EVC_KERNEL_CHECK();
    reg_final_kernel<<<1, 1024, 0, st>>>(partial, fx_data, limbs, nll_out, fx_out, dots);
    EVC_KERNEL_CHECK();
    return 0;
}

__global__ void dot_kernel(const float *__restrict__ a, const float *__restrict__ b, int64_t n,
                           double *__restrict__ partial)
{
    __shared__ double s_red[32];
    double acc = 0.0;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x)
        acc += (double)a[e] * (double)b[e];
    const double tot = cta_sum(acc, s_red);
    if (threadIdx.x == 0) partial[blockIdx.x] = tot;
}

// mode 0: out = sum; 1: out = sum / den[0]; 2: out = aux[0] - sum / den[0]
__global__ void __launch_bounds__(1024)
scalar_final_kernel(const double *__restrict__ partial, int mode, const double *__restrict__ den,
                    const double *__restrict__ aux, double *__restrict__ out)
{
    __shared__ double s_red[1024];
    const double v = final_sum(partial, s_red);
    if (threadIdx.x == 0) {
        if (mode == 0) out[0] = v;
        else if (mode == 1) out[0] = v / den[0];
        else out[0] = aux[0] - v / den[0];
    }
}

int vec_dot(const float *a, const float *b, int64_t n, double *out, double *partial, cudaStream_t st)
{
    dot_kernel<<<RED_BLOCKS, RED_THREADS, 0, st>>>(a, b, n, partial);
    EVC_KERNEL_CHECK();
    scalar_final_kernel<<<1, 1024, 0, st>>>(partial, 0, nullptr, nullptr, out);
    EVC_KERNEL_CHECK();
    return 0;
}

__global__ void axpby_kernel(float *__restrict__ y, const float *__restrict__ x, float a, float b, int64_t n)
{
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n;
         e += (int64_t)gridDim.x * blockDim.x)
        y[e] = b == 0.f ? a * x[e] : a * x[e] + b * y[e];
}

int vec_axpby(float *y, const float *x, float a, float b, int64_t n, cudaStream_t st)
{
    axpby_kernel<<<2048, 256, 0, st>>>(y, x, a, b, n);
    EVC_KERNEL_CHECK();
    return 0;
}

__global__ void sub_kernel(float *__restrict__ out, const float *__restrict__ a, const float *__restrict__ b,
                           int64_t n)
{
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n;
         e += (int64_t)gridDim.x * blockDim.x)
        out[e] = a[e] - b[e];
}

int vec_sub(float *out, const float *a, const float *b, int64_t n, cudaStream_t st)
{
    sub_kernel<<<2048, 256, 0, st>>>(out, a, b, n);
    EVC_KERNEL_CHECK();
    return 0;
}

// s = x - xp, y = g - gp; partials of y.s and y.y
__global__ void pair_update_kernel(float *__restrict__ s, float *__restrict__ y, const float *__restrict__ x,
                                   const float *__restrict__ xp, const float *__restrict__ g,
                                   const float *__restrict__ gp, int64_t n, double *__restrict__ partial)
{
    __shared__ double s_red[32];
    double ays = 0.0, ayy = 0.0;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        const float sv = x[e] - xp[e];
        const float yv = g[e] - gp[e];
        s[e] = sv;
        y[e] = yv;
        ays += (double)yv * (double)sv;
        ayy += (double)yv * (double)yv;
    }
    const double t0 = cta_sum(ays, s_red);
    const double t1 = cta_sum(ayy, s_red);
    if (threadIdx.x == 0) {
        partial[blockIdx.x] = t0;
        partial[RED_BLOCKS + blockIdx.x] = t1;
    }
}

int lbfgs_update_pair(float *s, float *y, const float *x, const float *xp, const float *g, const float *gp, double *ys,
                      double *yy, int64_t n, double *partial, cudaStream_t st)
{
    pair_update_kernel<<<RED_BLOCKS, RED_THREADS, 0, st>>>(s, y, x, xp, g, gp, n, partial);
    EVC_KERNEL_CHECK();
    scalar_final_kernel<<<1, 1024, 0, st>>>(partial, 0, nullptr, nullptr, ys);
    EVC_KERNEL_CHECK();
    scalar_final_kernel<<<1, 1024, 0, st>>>(partial + RED_BLOCKS, 0, nullptr, nullptr, yy);
    EVC_KERNEL_CHECK();
    return 0;
}

// two-loop building block:  d = (INIT ? -g : d + sign*coef[0]*v) * (num ? num[0]/den[0] : 1);  partial(u . d)
template <bool INIT>
__global__ void axpy_dot_kernel(float *__restrict__ d, const float *__restrict__ g_or_v,
                                const double *__restrict__ coef, float sign, const double *__restrict__ num,
                                const double *__restrict__ den, const float *__restrict__ u, int64_t n,
                                double *__restrict__ partial)
{
    __shared__ double s_red[32];
    const float c = INIT ? 0.f : sign * (float)coef[0];
    const float gamma = num != nullptr ? (float)(num[0] / den[0]) : 1.f;
    double acc = 0.0;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
        float dv = INIT ? -g_or_v[e] : fmaf(c, g_or_v[e], d[e]);
        dv *= gamma;
        d[e] = dv;
        if (u != nullptr) acc += (double)u[e] * (double)dv;
    }
    if (u != nullptr) {
        const double tot = cta_sum(acc, s_red);
        if (threadIdx.x == 0) partial[blockIdx.x] = tot;
    }
}

// Two-loop recursion (Nocedal), same ring-buffer convention as libLBFGS: `end` is the slot that will be written next,
// the `bound` most recent pairs precede it.
int lbfgs_direction(float *d, const float *g, const float *const *S, const float *const *Y, const double *ys,
                    double *alpha, double *coef, const double *yy, int64_t n, int m, int bound, int end,
                    double *partial, cudaStream_t st)
{
    if (bound == 0) {
        axpy_dot_kernel<true><<<RED_BLOCKS, RED_THREADS, 0, st>>>(d, g, nullptr, 0.f, nullptr, nullptr, nullptr, n,
                                                                 partial);
        EVC_KERNEL_CHECK();
        return 0;
    }
    const int newest = (end + m - 1) % m;
    int j = newest;
    // d = -g; alpha_newest = (s_newest . d) / ys
    axpy_dot_kernel<true><<<RED_BLOCKS, RED_THREADS, 0, st>>>(d, g, nullptr, 0.f, nullptr, nullptr, S[j], n, partial);
    EVC_KERNEL_CHECK();
    scalar_final_kernel<<<1, 1024, 0, st>>>(partial, 1, ys + j, nullptr, alpha + j);
    EVC_KERNEL_CHECK();
    for (int it = 0; it < bound; it++) {
        const bool last = it == bound - 1;
        if (!last) {
            const int jn = (j + m - 1) % m;
            // d -= alpha_j y_j; alpha_jn = (s_jn . d) / ys_jn
            axpy_dot_kernel<false><<<RED_BLOCKS, RED_THREADS, 0, st>>>(d, Y[j], alpha + j, -1.f, nullptr, nullptr,
                                                                      S[jn], n, partial);
            EVC_KERNEL_CHECK();
            scalar_final_kernel<<<1, 1024, 0, st>>>(partial, 1, ys + jn, nullptr, alpha + jn);
            EVC_KERNEL_CHECK();
            j = jn;
        } else {
            // oldest pair: d = (d - alpha_j y_j) * ys_newest / yy_newest; coef = alpha_j - (y_j . d) / ys_j
            axpy_dot_kernel<false><<<RED_BLOCKS, RED_THREADS, 0, st>>>(d, Y[j], alpha + j, -1.f, ys + newest, yy,
                                                                      Y[j], n, partial);
            EVC_KERNEL_CHECK();
            scalar_final_kernel<<<1, 1024, 0, st>>>(partial, 2, ys + j, alpha + j, coef);
            EVC_KERNEL_CHECK();
        }
    }
    for (int it = 0; it < bound; it++) {
        const bool last = it == bound - 1;
        const int jn = (j + 1) % m;
        // d += coef s_j; coef' = alpha_jn - (y_jn . d) / ys_jn
        axpy_dot_kernel<false><<<RED_BLOCKS, RED_THREADS, 0, st>>>(d, S[j], coef, 1.f, nullptr, nullptr,
                                                                  last ? nullptr : Y[jn], n, partial);
        EVC_KERNEL_CHECK();
        if (!last) {
            scalar_final_kernel<<<1, 1024, 0, st>>>(partial, 2, ys + jn, alpha + jn, coef);
            EVC_KERNEL_CHECK();
        }
        j = jn;
    }
    return 0;
}

// Checksum of a vector's bit patterns (evc_vec_checksum): the terms are summed modulo 2^64, an associative and
// commutative operation, so the integer atomics give the same value for every grid and every order.
__global__ void checksum_kernel(const unsigned int *__restrict__ v, int64_t n, unsigned long long *__restrict__ out)
{
    unsigned long long acc = 0ull;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x)
        acc += splitmix64_mix(((uint64_t)e + 1ull) * GOLDEN_GAMMA ^ (uint64_t)v[e]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0 && acc != 0ull) atomicAdd(out, acc);
}

int vec_checksum(const float *v, int64_t n, uint64_t *out, cudaStream_t st)
{
    if (!v || !out || n < 0) { set_error("evc_vec_checksum: bad arguments"); return 1; }
    EVC_CUDA(cudaMemsetAsync(out, 0, sizeof(uint64_t), st));
    if (n == 0) return 0;
    const int64_t blocks = std::min<int64_t>(1024, ceil_div(n, (int64_t)RED_THREADS));
    checksum_kernel<<<(unsigned)blocks, RED_THREADS, 0, st>>>(reinterpret_cast<const unsigned int *>(v), n,
                                                             reinterpret_cast<unsigned long long *>(out));
    EVC_KERNEL_CHECK();
    return 0;
}

// a10: Frobenius norm of every J block (raw gauge), one warp per pair
__global__ void fn_scores_kernel(const float *__restrict__ J, int64_t npairs, int qq, float *__restrict__ fn)
{
    const int64_t p = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (p >= npairs) return;
    const float *B = J + p * qq;
    double acc = 0.0;
    for (int e = lane; e < qq; e += 32) acc += (double)B[e] * (double)B[e];
    acc = warp_sum(acc);
    if (lane == 0) fn[p] = (float)sqrt(acc);
}

int fn_scores(const float *J, int L, int q, float *fn, cudaStream_t st)
{
    const int64_t npairs = (int64_t)L * (L - 1) / 2;
    if (npairs == 0) return 0;
    fn_scores_kernel<<<(unsigned)ceil_div(npairs, 8), 256, 0, st>>>(J, npairs, q * q, fn);
    EVC_KERNEL_CHECK();
    return 0;
}

}  // namespace evc
