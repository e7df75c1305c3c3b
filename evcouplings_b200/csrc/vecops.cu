// a8: device-side vector algebra for L-BFGS (SURVEY.md 8a row a8) and the EC Frobenius norms (a10).
// plmc drives libLBFGS on the host CPU; here the n-vector work (n = L*q + L(L-1)/2*q^2, 8.8M floats
// at L=200) stays in HBM and every scalar (dot products, alpha/beta of the two-loop recursion) stays
// on the device in double, so a direction costs no host round trip.  All reductions use a fixed grid
// and a fixed summation tree => bit-identical on every rank of a data-parallel run.
// These kernels are HBM-streaming: (4m+6)*n*4 bytes per iteration (SURVEY 8d).
#include <algorithm>
#include <map>
#include <mutex>
#include <utility>

#include "common.cuh"
#include "internal.h"

namespace evc {

constexpr int RED_BLOCKS = 1024;
constexpr int RED_THREADS = 256;

// Reduction partials are kept per (device, stream): two problems / threads / streams on one device no longer share
// a buffer (ADVICE r1).  Buffers live for the lifetime of the process (a few KB each).
static std::mutex g_scratch_mutex;
static std::map<std::pair<int, cudaStream_t>, double *> g_scratch;

double *reduction_scratch(int nd, cudaStream_t st)
{
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) {
        set_error("reduction_scratch: bad device");
        return nullptr;
    }
    if (nd > 4 * RED_BLOCKS) {
        set_error("reduction_scratch: request too large");
        return nullptr;
    }
    std::lock_guard<std::mutex> lock(g_scratch_mutex);
    double *&slot = g_scratch[std::make_pair(dev, st)];
    if (!slot && cudaMalloc(&slot, 4 * RED_BLOCKS * sizeof(double)) != cudaSuccess) {
        slot = nullptr;
        set_error("reduction_scratch: cudaMalloc failed");
        return nullptr;
    }
    return slot;
}

__device__ __forceinline__ double block_sum(double v, double *s_red)
{
    v = warp_sum(v);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s_red[warp] = v;
    __syncthreads();
    double tot = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) tot += s_red[w];
    __syncthreads();
    return tot;   // valid on thread 0
}

__global__ void dot_partial_kernel(const float *__restrict__ a, const float *__restrict__ b, int64_t n,
                                   double *__restrict__ partial)
{
    __shared__ double s_red[32];
    double acc = 0.0;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n;
         e += (int64_t)gridDim.x * blockDim.x)
        acc += (double)a[e] * (double)b[e];
    const double tot = block_sum(acc, s_red);
    if (threadIdx.x == 0) partial[blockIdx.x] = tot;
}

// mode 0: out = sum; 1: out = sum / den; 2: out = aux - sum / den
__global__ void reduce_final_kernel(const double *__restrict__ partial, int nblocks, int mode,
                                    const double *__restrict__ den, const double *__restrict__ aux,
                                    double *__restrict__ out)
{
    __shared__ double s_red[RED_BLOCKS];
    const int tid = threadIdx.x;
    s_red[tid] = tid < nblocks ? partial[tid] : 0.0;
    __syncthreads();
    for (int o = RED_BLOCKS / 2; o > 0; o >>= 1) {
        if (tid < o) s_red[tid] += s_red[tid + o];
        __syncthreads();
    }
    if (tid == 0) {
        double v = s_red[0];
        if (mode == 1) v = v / den[0];
        else if (mode == 2) v = aux[0] - v / den[0];
        out[0] = v;
    }
}

static int dot_mode(const float *a, const float *b, int64_t n, int mode, const double *den,
                    const double *aux, double *out, cudaStream_t st)
{
    double *partial = reduction_scratch(RED_BLOCKS, st);
    if (!partial) return 1;
    dot_partial_kernel<<<RED_BLOCKS, RED_THREADS, 0, st>>>(a, b, n, partial);
    EVC_KERNEL_CHECK();
    reduce_final_kernel<<<1, RED_BLOCKS, 0, st>>>(partial, RED_BLOCKS, mode, den, aux, out);
    EVC_KERNEL_CHECK();
    return 0;
}

int vec_dot(const float *a, const float *b, int64_t n, double *out, cudaStream_t st)
{
    return dot_mode(a, b, n, 0, nullptr, nullptr, out, st);
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

// y += sign * coef[0] * x   (coef lives on the device)
__global__ void axpy_dev_kernel(float *__restrict__ y, const float *__restrict__ x,
                                const double *__restrict__ coef, float sign, int64_t n)
{
    const float c = sign * (float)coef[0];
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n;
         e += (int64_t)gridDim.x * blockDim.x)
        y[e] += c * x[e];
}

// y *= num[0] / den[0]
__global__ void scale_dev_kernel(float *__restrict__ y, const double *__restrict__ num,
                                 const double *__restrict__ den, int64_t n)
{
    const float c = (float)(num[0] / den[0]);
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n;
         e += (int64_t)gridDim.x * blockDim.x)
        y[e] *= c;
}

// Two-loop recursion (Nocedal), same ring-buffer convention as libLBFGS: `end` is the slot that
// will be written next, the `bound` most recent pairs precede it.
// scratch: [0] = y.y of the newest pair, [1] = temp, [2 .. 2+m) = alpha per slot.
int lbfgs_direction(float *d, const float *g, const float *S, const float *Y, const double *ys,
                    double *scratch, int64_t n, int m, int bound, int end, cudaStream_t st)
{
    if (bound > m || bound < 0 || m <= 0) { set_error("lbfgs_direction: bad history bounds"); return 1; }
    if (vec_axpby(d, g, -1.f, 0.f, n, st)) return 1;
    if (bound == 0) return 0;
    double *alpha = scratch + 2;
    int j = end;
    for (int it = 0; it < bound; it++) {
        j = (j + m - 1) % m;
        // alpha_j = (s_j . d) / ys_j ;  d -= alpha_j y_j
        if (dot_mode(S + (int64_t)j * n, d, n, 1, ys + j, nullptr, alpha + j, st)) return 1;
        axpy_dev_kernel<<<2048, 256, 0, st>>>(d, Y + (int64_t)j * n, alpha + j, -1.f, n);
        EVC_KERNEL_CHECK();
    }
    const int last = (end + m - 1) % m;
    scale_dev_kernel<<<2048, 256, 0, st>>>(d, ys + last, scratch + 0, n);
    EVC_KERNEL_CHECK();
    for (int it = 0; it < bound; it++) {
        // beta = (y_j . d) / ys_j ;  d += (alpha_j - beta) s_j
        if (dot_mode(Y + (int64_t)j * n, d, n, 2, ys + j, alpha + j, scratch + 1, st)) return 1;
        axpy_dev_kernel<<<2048, 256, 0, st>>>(d, S + (int64_t)j * n, scratch + 1, 1.f, n);
        EVC_KERNEL_CHECK();
        j = (j + 1) % m;
    }
    return 0;
}

__global__ void update_pair_kernel(float *__restrict__ s, float *__restrict__ y, const float *__restrict__ x,
                                   const float *__restrict__ xp, const float *__restrict__ g,
                                   const float *__restrict__ gp, int64_t n, double *__restrict__ partial)
{
    __shared__ double s_red[32];
    double ays = 0.0, ayy = 0.0;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n;
         e += (int64_t)gridDim.x * blockDim.x) {
        const float sv = x[e] - xp[e];
        const float yv = g[e] - gp[e];
        s[e] = sv;
        y[e] = yv;
        ays += (double)yv * (double)sv;
        ayy += (double)yv * (double)yv;
    }
    const double t0 = block_sum(ays, s_red);
    const double t1 = block_sum(ayy, s_red);
    if (threadIdx.x == 0) {
        partial[blockIdx.x] = t0;
        partial[RED_BLOCKS + blockIdx.x] = t1;
    }
}

int lbfgs_update_pair(float *s, float *y, const float *x, const float *xp, const float *g,
                      const float *gp, double *ys, double *yy, int64_t n, cudaStream_t st)
{
    double *partial = reduction_scratch(2 * RED_BLOCKS, st);
    if (!partial) return 1;
    update_pair_kernel<<<RED_BLOCKS, RED_THREADS, 0, st>>>(s, y, x, xp, g, gp, n, partial);
    EVC_KERNEL_CHECK();
    reduce_final_kernel<<<1, RED_BLOCKS, 0, st>>>(partial, RED_BLOCKS, 0, nullptr, nullptr, ys);
    EVC_KERNEL_CHECK();
    reduce_final_kernel<<<1, RED_BLOCKS, 0, st>>>(partial + RED_BLOCKS, RED_BLOCKS, 0, nullptr, nullptr, yy);
    EVC_KERNEL_CHECK();
    return 0;
}

// Checksum of a vector's bit patterns (evc_vec_checksum): the terms are summed modulo 2^64, an associative and
// commutative operation, so the integer atomics give the same value for every grid and every order.
__device__ __forceinline__ unsigned long long checksum_mix(unsigned long long i, unsigned int bits)
{
    unsigned long long z = ((i + 1ull) * 0x9E3779B97F4A7C15ull) ^ (unsigned long long)bits;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

__global__ void checksum_kernel(const unsigned int *__restrict__ v, int64_t n, unsigned long long *__restrict__ out)
{
    unsigned long long acc = 0ull;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x)
        acc += checksum_mix((unsigned long long)e, v[e]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0 && acc != 0ull) atomicAdd(out, acc);
}

int vec_checksum(const float *v, int64_t n, uint64_t *out, cudaStream_t st)
{
    if (!v || !out || n < 0) { set_error("evc_vec_checksum: bad arguments"); return 1; }
    EVC_CUDA(cudaMemsetAsync(out, 0, sizeof(uint64_t), st));
    if (n == 0) return 0;
    const int64_t blocks = std::min<int64_t>(RED_BLOCKS, ceil_div(n, (int64_t)RED_THREADS));
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
