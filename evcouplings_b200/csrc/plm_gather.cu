// Hot path (a): pseudo-likelihood objective + gradient, gather/scatter formulation (sm_90a).
// (First correct CUDA path and the measured comparison baseline of the tensor-core path in plm_tc.cu; still
//  used for f_i / f_ij counting, the statistical energies, and selectable with forward/backward = "gather".)
//
// Replaces the inner loop of plmc's L-BFGS (SURVEY.md 8a row a7; reference call
// site evcouplings/couplings/tools.py:202-266): for every sequence n and site i
//     z_a = h_i(a) + sum_{j != i} J_ij(a, s_nj);  P = softmax(z)
//     fx -= w_n log P[s_ni];   r_a = w_n (P_a - [a = s_ni])
//     g_h[i][a] += r_a;        g_J[i,j][a][s_nj] += r_a   for every j != i
// and the symmetric J_ij is shared by conditionals i and j.
//
// HBM layouts (all fp32 unless noted)
//   x      [h : L*q | J : L(L-1)/2 * q*q]          parameters, plmc .model order
//   W      [L][Lp][QB][S]   expanded couplings, W[i][j][b][a] = J_ij(a,b); a fastest,
//          odd row stride S so that 32 threads gathering rows b_0..b_31 of one (i,j)
//          block hit 32 different shared-memory banks; block (i,i), padded sites
//          j >= L and (ignore_gaps) the gap row b = q are zero => no branches in the loop
//   msa4   [Lp/4][Nld] uint32, four consecutive sites of one sequence per word,
//          sequence index fastest (a warp reads 128 contiguous bytes)
//   R      [L][Nr][S]       residuals r for conditional i (written by forward,
//          bulk-copied as one contiguous tile by backward)
//   perm   [ntiles_b][L][2224] uint32 byte offsets of the tile's residual rows, grouped by the
//          sequence's state at column j, buckets 8-aligned and padded with a zero row;
//          bstart [ntiles_b][L][24] uint16 bucket boundaries (static per MSA)
//   G      same geometry as W: G[i][j][b][a] = sum_n r_ni(a) [s_nj = b]
//
// Kernels
//   plm_expand     x -> W (both orientations of every block)
//   plm_fwd        thread = sequence, CTA = (512 sequences, site i); the 353 KB row block
//                  W[i] streams through shared memory in 24-site chunks with
//                  cp.async.bulk (TMA 1-D) + mbarrier double buffering; 21 accumulators
//                  per sequence in registers; softmax in registers; writes R, per-CTA
//                  partials of g_h and fx (deterministic two-stage reduction)
//   plm_bwd        CTA = (2048-sequence tile, site i): R tile (172 KB) bulk-copied to shared
//                  memory; warp = column j, lane = state a; every (j, b) bucket is a
//                  branch-free register accumulation of shared-memory rows
//                  (LDG.128 of 4 offsets -> 4 x (IADD, LDS, FADD)), one RED per bucket
//   plm_finalize   g_J(i<j)[a][b] = G[i][j][b][a] + G[j][i][a][b]; g_h, fx from partials
//
// Bound: on-chip.  Per cell-op (n,i,j,a) the path does one 4-byte shared-memory read
// in forward and one in backward; compulsory HBM traffic is ~1.9 GB / evaluation at
// N=50k, L=200 (R write+read, W, G), i.e. <1 ms of the measured 6.5 TB/s.
#include <cuda_bf16.h>

#include "common.cuh"
#include "internal.h"

namespace evc {

constexpr int FWD_JC = 24;        // sites per streamed chunk of W[i]
constexpr int FWD_THREADS = 256;
constexpr int BWD_THREADS = 1024;

bool plm_supported_q(int q, int gap_code)
{
    // every code, the ignored gap's included, must fit the 5 Hamming bit-planes (codes < 32)
    return q >= 2 && q <= PLM_MAX_Q && (gap_code < 0 || q <= PLM_MAX_Q - 1);
}

bool plm_gather_supported_q(int q) { return q == 21 || q == 20 || q == 5 || q == 4; }

// ----------------------------------------------------------------------------------------------
// one-time packing
// ----------------------------------------------------------------------------------------------
__global__ void pack_msa_kernel(const uint8_t *__restrict__ codes, uint32_t *__restrict__ msa4,
                                int64_t N, int L, int64_t Nld)
{
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int w = blockIdx.y;
    if (n >= Nld) return;
    uint32_t v = 0;
    if (n < N) {
#pragma unroll
        for (int u = 0; u < 4; u++) {
            const int site = w * 4 + u;
            const uint32_t c = site < L ? codes[n * L + site] : 0u;
            v |= c << (8 * u);
        }
    }
    msa4[(int64_t)w * Nld + n] = v;
}

int plm_pack_msa(const PlmGeom &g, const uint8_t *d_codes, uint32_t *d_msa4, cudaStream_t st)
{
    dim3 grid((unsigned)ceil_div(g.Nld, 256), (unsigned)(g.Lp / 4));
    pack_msa_kernel<<<grid, 256, 0, st>>>(d_codes, d_msa4, g.N, g.L, g.Nld);
    EVC_KERNEL_CHECK();
    return 0;
}

// state-sorted sequence lists per (backward tile, column): stable counting sort by one warp.
// Output per (tile, column): PLM_BWD_CAP uint32 byte offsets (row * S * 4) into the shared-memory residual
// tile, grouped by state; every bucket starts at a multiple of 8 entries and is padded with the offset of
// an all-zero row, so the consumer loop is branch-free.  bstart[b] .. bstart[b+1] (uint16, PLM_BWD_BS per
// list) delimit bucket b; ignored-gap sequences are not listed at all.
__global__ void build_buckets_kernel(const uint8_t *__restrict__ codes, uint32_t *__restrict__ perm,
                                     uint16_t *__restrict__ bstart, int64_t N, int L, int q, int S)
{
    __shared__ int hist[32];
    __shared__ int start[33];
    const int t = blockIdx.x, j = blockIdx.y, lane = threadIdx.x;
    const int64_t base = (int64_t)t * PLM_BWD_TS;
    const int cnt = (int)min((int64_t)PLM_BWD_TS, N - base);
    const int cnt32 = (cnt + 31) & ~31;
    uint32_t *out = perm + ((int64_t)t * L + j) * PLM_BWD_CAP;
    uint16_t *bs = bstart + ((int64_t)t * L + j) * PLM_BWD_BS;
    const uint32_t zero_off = (uint32_t)(PLM_BWD_TS * S * sizeof(float));
    hist[lane] = 0;
    __syncwarp();
    for (int k = lane; k < cnt32; k += 32) {
        int c = 31;
        if (k < cnt) {
            c = codes[(base + k) * L + j];
            if (c >= q) c = 31;            // ignored gap -> not listed
        }
        const unsigned m = __match_any_sync(0xffffffffu, c);
        if (lane == __ffs(m) - 1) hist[c] += __popc(m);
        __syncwarp();
    }
    // exclusive scan of the 8-aligned bucket sizes (lane = bucket); bucket 31 is dropped
    const int v = (lane < q) ? ((hist[lane] + 7) & ~7) : 0;
    int incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += u;
    }
    __syncwarp();
    start[lane] = incl - v;
    if (lane == 31) start[32] = incl;
    __syncwarp();
    if (lane <= q && lane < PLM_BWD_BS) bs[lane] = (uint16_t)start[lane < q ? lane : q];
    if (lane == 0) bs[q] = (uint16_t)start[q];
    // pad slots first (zero-row offset), then scatter the real entries
    for (int b = 0; b < q; b++) {
        const int s0 = start[b] + hist[b], s1 = start[b] + ((hist[b] + 7) & ~7);
        for (int k = s0 + lane; k < s1; k += 32) out[k] = zero_off;
    }
    __syncwarp();
    hist[lane] = start[lane];            // running write positions
    __syncwarp();
    for (int k = lane; k < cnt32; k += 32) {
        int c = 31;
        if (k < cnt) {
            c = codes[(base + k) * L + j];
            if (c >= q) c = 31;
        }
        const unsigned m = __match_any_sync(0xffffffffu, c);
        const int pos = hist[c] + __popc(m & ((1u << lane) - 1u));
        __syncwarp();
        if (lane == __ffs(m) - 1) hist[c] += __popc(m);
        __syncwarp();
        if (c < q) out[pos] = (uint32_t)(k * S * sizeof(float));
    }
}

int plm_build_buckets(const PlmGeom &g, const uint8_t *d_codes, uint32_t *d_perm, uint16_t *d_bstart,
                      cudaStream_t st)
{
    dim3 grid((unsigned)g.ntiles_b, (unsigned)g.L);
    build_buckets_kernel<<<grid, 32, 0, st>>>(d_codes, d_perm, d_bstart, g.N, g.L, g.q, g.S);
    EVC_KERNEL_CHECK();
    return 0;
}

// ----------------------------------------------------------------------------------------------
// expand: x (tri blocks [a][b]) -> W[i][j][b][a] and W[j][i][a][b]
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ int64_t pair_index(int i, int j, int L)
{
    return (int64_t)i * (2 * L - i - 1) / 2 + (j - i - 1);
}

__global__ void expand_kernel(const float *__restrict__ x, float *__restrict__ W, int L, int Lp, int q,
                              int QB, int S)
{
    const int i = blockIdx.y, j = blockIdx.x;
    if (j <= i) return;
    const float *J = x + (int64_t)L * q + pair_index(i, j, L) * q * q;
    const int64_t blk = (int64_t)QB * S;
    float *Wij = W + ((int64_t)i * Lp + j) * blk;
    float *Wji = W + ((int64_t)j * Lp + i) * blk;
    for (int e = threadIdx.x; e < q * q; e += blockDim.x) {
        const int a = e / q, b = e - a * q;
        const float v = J[e];
        Wij[b * S + a] = v;
        Wji[a * S + b] = v;
    }
}

int plm_expand(const PlmGeom &g, const float *d_x, float *d_W, cudaStream_t st)
{
    dim3 grid((unsigned)g.L, (unsigned)g.L);
    expand_kernel<<<grid, 128, 0, st>>>(d_x, d_W, g.L, g.Lp, g.q, g.QB, g.S);
    EVC_KERNEL_CHECK();
    return 0;
}

// ----------------------------------------------------------------------------------------------
// forward: logits, softmax, residuals
// ----------------------------------------------------------------------------------------------
template <int Q, int S>
__global__ void __launch_bounds__(FWD_THREADS, 2)
plm_fwd_kernel(const float *__restrict__ W, const float *__restrict__ h,
               const uint32_t *__restrict__ msa4, const float *__restrict__ wts,
               float *__restrict__ R, __nv_bfloat16 *__restrict__ Rt_hi, __nv_bfloat16 *__restrict__ Rt_lo,
               int64_t Kp, float *__restrict__ gh_part, double *__restrict__ fx_part, PlmGeom g)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int BLK = g.QB * S;
    const int chunk_floats = FWD_JC * BLK;
    float *buf0 = reinterpret_cast<float *>(smem_raw);
    float *buf1 = buf0 + chunk_floats;
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + (size_t)2 * chunk_floats * sizeof(float));
    float *s_gh = reinterpret_cast<float *>(bars + 2);               // [8 warps][32]
    double *s_fx = reinterpret_cast<double *>(s_gh + 8 * 32);        // [8]

    const int tile = blockIdx.x, i = blockIdx.y;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t N = g.N;
    const int64_t n0 = (int64_t)tile * PLM_FWD_TS + tid;
    const int64_t n1 = n0 + FWD_THREADS;
    const int64_t m0 = n0 < N ? n0 : N - 1;
    const int64_t m1 = n1 < N ? n1 : N - 1;
    const int Lp = g.Lp;
    const int nchunks = (Lp + FWD_JC - 1) / FWD_JC;
    const float *Wi = W + (int64_t)i * g.row_block();

    if (tid == 0) {
        mbar_init(&bars[0], 1);
        mbar_init(&bars[1], 1);
        mbar_fence_init();
    }
    __syncthreads();
    if (tid == 0) {
        const uint32_t bytes = (uint32_t)(min(FWD_JC, Lp) * BLK * sizeof(float));
        mbar_expect_tx(&bars[0], bytes);
        bulk_g2s(buf0, Wi, bytes, &bars[0]);
    }

    float z0[Q], z1[Q];
#pragma unroll
    for (int a = 0; a < Q; a++) { z0[a] = 0.f; z1[a] = 0.f; }

    for (int c = 0; c < nchunks; c++) {
        const int j0 = c * FWD_JC;
        const int jc = min(FWD_JC, Lp - j0);
        if (tid == 0 && c + 1 < nchunks) {
            const int jn = min(FWD_JC, Lp - (j0 + FWD_JC));
            const uint32_t bytes = (uint32_t)(jn * BLK * sizeof(float));
            uint64_t *bar = &bars[(c + 1) & 1];
            mbar_expect_tx(bar, bytes);
            bulk_g2s(((c + 1) & 1) ? buf1 : buf0, Wi + (int64_t)(j0 + FWD_JC) * BLK, bytes, bar);
        }
        uint32_t pk0[FWD_JC / 4], pk1[FWD_JC / 4];
#pragma unroll
        for (int u = 0; u < FWD_JC / 4; u++) {
            pk0[u] = 0; pk1[u] = 0;
            if (u * 4 < jc) {
                const int64_t off = (int64_t)(j0 / 4 + u) * g.Nld;
                pk0[u] = msa4[off + m0];
                pk1[u] = msa4[off + m1];
            }
        }
        mbar_wait(&bars[c & 1], (uint32_t)((c >> 1) & 1));
        const float *B = (c & 1) ? buf1 : buf0;
#pragma unroll
        for (int u = 0; u < FWD_JC / 4; u++) {
            if (u * 4 < jc) {
#pragma unroll
                for (int v = 0; v < 4; v++) {
                    const int jj = u * 4 + v;
                    const uint32_t b0 = (pk0[u] >> (8 * v)) & 0xffu;
                    const uint32_t b1 = (pk1[u] >> (8 * v)) & 0xffu;
                    const float *c0 = B + jj * BLK + b0 * S;
                    const float *c1 = B + jj * BLK + b1 * S;
#pragma unroll
                    for (int a = 0; a < Q; a++) {
                        z0[a] += c0[a];
                        z1[a] += c1[a];
                    }
                }
            }
        }
        __syncthreads();   // buffer (c & 1) is free for the copy issued at iteration c + 1
    }

    // ---- softmax + residuals, in registers ----------------------------------------------
    const uint32_t wi0 = msa4[(int64_t)(i >> 2) * g.Nld + m0];
    const uint32_t wi1 = msa4[(int64_t)(i >> 2) * g.Nld + m1];
    const int si0 = (int)((wi0 >> (8 * (i & 3))) & 0xffu);
    const int si1 = (int)((wi1 >> (8 * (i & 3))) & 0xffu);
    const float w0 = (n0 < N && si0 < Q) ? wts[m0] : 0.f;
    const float w1 = (n1 < N && si1 < Q) ? wts[m1] : 0.f;

    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int a = 0; a < Q; a++) {
        const float hv = h[i * Q + a];
        z0[a] += hv; z1[a] += hv;
        mx0 = fmaxf(mx0, z0[a]); mx1 = fmaxf(mx1, z1[a]);
    }
    float zs0 = 0.f, zs1 = 0.f, sum0 = 0.f, sum1 = 0.f;
#pragma unroll
    for (int a = 0; a < Q; a++) {
        if (a == si0) zs0 = z0[a];
        if (a == si1) zs1 = z1[a];
        z0[a] = expf(z0[a] - mx0); sum0 += z0[a];
        z1[a] = expf(z1[a] - mx1); sum1 += z1[a];
    }
    const float lp0 = zs0 - mx0 - logf(sum0);
    const float lp1 = zs1 - mx1 - logf(sum1);
    double fx_local = -((double)w0 * (double)lp0 + (double)w1 * (double)lp1);
    if (w0 == 0.f && w1 == 0.f) fx_local = 0.0;
    else if (w0 == 0.f) fx_local = -((double)w1 * (double)lp1);
    else if (w1 == 0.f) fx_local = -((double)w0 * (double)lp0);
    const float inv0 = w0 / sum0, inv1 = w1 / sum1;
#pragma unroll
    for (int a = 0; a < Q; a++) {
        z0[a] = z0[a] * inv0 - (a == si0 ? w0 : 0.f);
        z1[a] = z1[a] * inv1 - (a == si1 ? w1 : 0.f);
    }
    if (Rt_hi != nullptr) {
        // tensor-core backward: residuals transposed (sequence index fastest => coalesced), split in two bf16
#pragma unroll
        for (int a = 0; a < Q; a++) {
            const int64_t rowoff = ((int64_t)i * Q + a) * Kp;
            if (n0 < N) {
                const __nv_bfloat16 hi = __float2bfloat16_rn(z0[a]);
                Rt_hi[rowoff + n0] = hi;
                Rt_lo[rowoff + n0] = __float2bfloat16_rn(z0[a] - __bfloat162float(hi));
            }
            if (n1 < N) {
                const __nv_bfloat16 hi = __float2bfloat16_rn(z1[a]);
                Rt_hi[rowoff + n1] = hi;
                Rt_lo[rowoff + n1] = __float2bfloat16_rn(z1[a] - __bfloat162float(hi));
            }
        }
    } else {
        if (n0 < N) {
            float *r = R + ((int64_t)i * g.Nr + n0) * S;
#pragma unroll
            for (int a = 0; a < S; a++) r[a] = a < Q ? z0[a < Q ? a : 0] : 0.f;
        }
        if (n1 < N) {
            float *r = R + ((int64_t)i * g.Nr + n1) * S;
#pragma unroll
            for (int a = 0; a < S; a++) r[a] = a < Q ? z1[a < Q ? a : 0] : 0.f;
        }
    }
    // deterministic CTA reduction of g_h and fx
#pragma unroll
    for (int a = 0; a < Q; a++) {
        const float v = warp_sum(z0[a] + z1[a]);
        if (lane == 0) s_gh[warp * 32 + a] = v;
    }
    const double fw = warp_sum(fx_local);
    if (lane == 0) s_fx[warp] = fw;
    __syncthreads();
    if (tid < S) {
        float tot = 0.f;
        if (tid < Q)
            for (int w = 0; w < FWD_THREADS / 32; w++) tot += s_gh[w * 32 + tid];
        gh_part[((int64_t)i * g.ntiles_f + tile) * S + tid] = tot;
    }
    if (tid == 0) {
        double tot = 0.0;
        for (int w = 0; w < FWD_THREADS / 32; w++) tot += s_fx[w];
        fx_part[(int64_t)i * g.ntiles_f + tile] = tot;
    }
}

static size_t fwd_smem_bytes(const PlmGeom &g)
{
    return (size_t)2 * FWD_JC * g.QB * g.S * sizeof(float) + 2 * sizeof(uint64_t) +
           8 * 32 * sizeof(float) + 8 * sizeof(double);
}

template <int Q, int S>
static int launch_fwd(const PlmGeom &g, const float *W, const float *x, const uint32_t *msa4,
                      const float *wts, float *R, void *rt_hi, void *rt_lo, int64_t Kp, float *gh_part,
                      double *fx_part, cudaStream_t st)
{
    const size_t smem = fwd_smem_bytes(g);
    EVC_CUDA(cudaFuncSetAttribute(plm_fwd_kernel<Q, S>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)smem));
    dim3 grid((unsigned)g.ntiles_f, (unsigned)g.L);
    plm_fwd_kernel<Q, S><<<grid, FWD_THREADS, smem, st>>>(W, x, msa4, wts, R,
                                                          reinterpret_cast<__nv_bfloat16 *>(rt_hi),
                                                          reinterpret_cast<__nv_bfloat16 *>(rt_lo), Kp, gh_part,
                                                          fx_part, g);
    EVC_KERNEL_CHECK();
    return 0;
}

int plm_forward(const PlmGeom &g, const float *d_W, const float *d_x, const uint32_t *d_msa4,
                const float *d_wts, float *d_R, void *d_rt_hi, void *d_rt_lo, int64_t Kp, float *d_gh_part,
                double *d_fx_part, cudaStream_t st)
{
#define EVC_FWD(QQ, SS) \
    return launch_fwd<QQ, SS>(g, d_W, d_x, d_msa4, d_wts, d_R, d_rt_hi, d_rt_lo, Kp, d_gh_part, d_fx_part, st)
    switch (g.q) {
        case 21: EVC_FWD(21, 21);
        case 20: EVC_FWD(20, 21);
        case 5: EVC_FWD(5, 5);
        case 4: EVC_FWD(4, 5);
    }
#undef EVC_FWD
    set_error("plm_forward: unsupported number of states q=" + std::to_string(g.q));
    return 1;
}

// R = w * onehot (for the weighted pair counts f_ij); same grid as forward
__global__ void onehot_residual_kernel(const uint32_t *__restrict__ msa4, const float *__restrict__ wts,
                                       float *__restrict__ R, float *__restrict__ gh_part, PlmGeom g)
{
    __shared__ float s_gh[8 * 32];
    const int tile = blockIdx.x, i = blockIdx.y;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int Q = g.q, S = g.S;
    float acc[2] = {0.f, 0.f};
    int code[2] = {255, 255};
    for (int u = 0; u < 2; u++) {
        const int64_t n = (int64_t)tile * PLM_FWD_TS + tid + u * FWD_THREADS;
        if (n < g.N) {
            const uint32_t wv = msa4[(int64_t)(i >> 2) * g.Nld + n];
            const int s = (int)((wv >> (8 * (i & 3))) & 0xffu);
            const float w = s < Q ? wts[n] : 0.f;
            float *r = R + ((int64_t)i * g.Nr + n) * S;
            for (int a = 0; a < S; a++) r[a] = (a == s) ? w : 0.f;
            acc[u] = w;
            code[u] = s;
        }
    }
    for (int a = 0; a < Q; a++) {
        const float v = warp_sum((code[0] == a ? acc[0] : 0.f) + (code[1] == a ? acc[1] : 0.f));
        if (lane == 0) s_gh[warp * 32 + a] = v;
    }
    __syncthreads();
    if (tid < S) {
        float tot = 0.f;
        if (tid < Q)
            for (int w = 0; w < FWD_THREADS / 32; w++) tot += s_gh[w * 32 + tid];
        gh_part[((int64_t)i * g.ntiles_f + tile) * S + tid] = tot;
    }
}

int plm_onehot_residual(const PlmGeom &g, const uint32_t *d_msa4, const float *d_wts, float *d_R,
                        float *d_gh_part, cudaStream_t st)
{
    dim3 grid((unsigned)g.ntiles_f, (unsigned)g.L);
    onehot_residual_kernel<<<grid, FWD_THREADS, 0, st>>>(d_msa4, d_wts, d_R, d_gh_part, g);
    EVC_KERNEL_CHECK();
    return 0;
}

// ----------------------------------------------------------------------------------------------
// backward: G[i][j][b][a] = sum over the (j,b) bucket of R_i[n][a]
// ----------------------------------------------------------------------------------------------
template <int S>
__global__ void __launch_bounds__(BWD_THREADS, 1)
plm_bwd_kernel(const float *__restrict__ R, const uint32_t *__restrict__ perm,
               const uint16_t *__restrict__ bstart, float *__restrict__ G, PlmGeom g)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float *Rs = reinterpret_cast<float *>(smem_raw);                       // [PLM_BWD_TS + 1][S]
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem_raw + (size_t)(PLM_BWD_TS + 4) * S * sizeof(float));
    int *s_next = reinterpret_cast<int *>(bar + 1);                        // dynamic column scheduler

    const int t = blockIdx.x, i = blockIdx.y;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t base = (int64_t)t * PLM_BWD_TS;
    const int cnt = (int)min((int64_t)PLM_BWD_TS, g.N - base);
    const int cnt4 = (cnt + 3) & ~3;
    const int Q = g.q;
    const int BLK = g.QB * S;

    if (tid == 0) {
        mbar_init(bar, 1);
        mbar_fence_init();
        *s_next = BWD_THREADS / 32;
    }
    if (tid < S) Rs[PLM_BWD_TS * S + tid] = 0.f;          // the all-zero row that padding entries point at
    __syncthreads();
    if (tid == 0) {
        const uint32_t bytes = (uint32_t)((size_t)cnt4 * S * sizeof(float));
        mbar_expect_tx(bar, bytes);
        bulk_g2s(Rs, R + ((int64_t)i * g.Nr + base) * S, bytes, bar);
    }
    mbar_wait(bar, 0);

    const char *Rl = reinterpret_cast<const char *>(Rs + (lane < S ? lane : 0));
    for (int j = warp; j < g.L;) {
        if (j == i) {
            int nj = 0;
            if (lane == 0) nj = atomicAdd(s_next, 1);
            j = __shfl_sync(0xffffffffu, nj, 0);
            continue;
        }
        const uint32_t *list = perm + ((int64_t)t * g.L + j) * PLM_BWD_CAP;
        const uint16_t *bs = bstart + ((int64_t)t * g.L + j) * PLM_BWD_BS;
        float *Gij = G + (int64_t)i * g.row_block() + (int64_t)j * BLK;
        const int my_start = (lane <= Q) ? (int)bs[lane] : 0;       // lane b holds bstart[b]
        for (int b = 0; b < Q; b++) {
            const int k0 = __shfl_sync(0xffffffffu, my_start, b);
            const int k1 = __shfl_sync(0xffffffffu, my_start, b + 1);
            if (k0 == k1) continue;
            float acc0 = 0.f, acc1 = 0.f;
            for (int k = k0; k < k1; k += 8) {
                const uint4 e0 = __ldg(reinterpret_cast<const uint4 *>(list + k));
                const uint4 e1 = __ldg(reinterpret_cast<const uint4 *>(list + k + 4));
                const float v0 = *reinterpret_cast<const float *>(Rl + e0.x);
                const float v1 = *reinterpret_cast<const float *>(Rl + e0.y);
                const float v2 = *reinterpret_cast<const float *>(Rl + e0.z);
                const float v3 = *reinterpret_cast<const float *>(Rl + e0.w);
                const float v4 = *reinterpret_cast<const float *>(Rl + e1.x);
                const float v5 = *reinterpret_cast<const float *>(Rl + e1.y);
                const float v6 = *reinterpret_cast<const float *>(Rl + e1.z);
                const float v7 = *reinterpret_cast<const float *>(Rl + e1.w);
                acc0 += (v0 + v1) + (v2 + v3);
                acc1 += (v4 + v5) + (v6 + v7);
            }
            if (lane < Q) atomicAdd(Gij + b * S + lane, acc0 + acc1);
        }
        int nj = 0;
        if (lane == 0) nj = atomicAdd(s_next, 1);      // next unclaimed column
        j = __shfl_sync(0xffffffffu, nj, 0);
    }
}

int plm_backward(const PlmGeom &g, const float *d_R, const uint32_t *d_perm, const uint16_t *d_bstart,
                 float *d_G, cudaStream_t st)
{
    dim3 grid((unsigned)g.ntiles_b, (unsigned)g.L);
    if (g.S == 21) {
        const size_t smem = (size_t)(PLM_BWD_TS + 4) * 21 * sizeof(float) + 2 * sizeof(uint64_t);
        EVC_CUDA(cudaFuncSetAttribute(plm_bwd_kernel<21>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)smem));
        plm_bwd_kernel<21><<<grid, BWD_THREADS, smem, st>>>(d_R, d_perm, d_bstart, d_G, g);
    } else if (g.S == 5) {
        const size_t smem = (size_t)(PLM_BWD_TS + 4) * 5 * sizeof(float) + 2 * sizeof(uint64_t);
        plm_bwd_kernel<5><<<grid, BWD_THREADS, smem, st>>>(d_R, d_perm, d_bstart, d_G, g);
    } else {
        set_error("plm_backward: unsupported row stride");
        return 1;
    }
    EVC_KERNEL_CHECK();
    return 0;
}

// ----------------------------------------------------------------------------------------------
// finalize: symmetrise G into the tri-block gradient; reduce g_h / fx partials
// ----------------------------------------------------------------------------------------------
__global__ void finalize_pairs_kernel(const float *__restrict__ G, float *__restrict__ gJ, int L, int Lp,
                                      int q, int QB, int S, float scale)
{
    const int i = blockIdx.y, j = blockIdx.x;
    if (j <= i) return;
    const int64_t blk = (int64_t)QB * S;
    const float *Gij = G + ((int64_t)i * Lp + j) * blk;   // [b][a]
    const float *Gji = G + ((int64_t)j * Lp + i) * blk;   // [a][b]
    float *out = gJ + pair_index(i, j, L) * q * q;
    for (int e = threadIdx.x; e < q * q; e += blockDim.x) {
        const int a = e / q, b = e - a * q;
        out[e] = scale * (Gij[b * S + a] + Gji[a * S + b]);
    }
}

__global__ void finalize_fields_kernel(const float *__restrict__ gh_part, const double *__restrict__ fx_part,
                                       float *__restrict__ gh, double *__restrict__ fx, int L, int q, int S,
                                       int ntiles)
{
    // blocks 0..L-1: g_h of site i (fixed summation order over tiles => deterministic);
    // block L: fx = sum of all per-CTA partials (fixed tree)
    __shared__ double s_red[256];
    const int tid = threadIdx.x;
    if ((int)blockIdx.x < L) {
        const int i = blockIdx.x;
        // 8 partial sums per state, combined in a fixed order
        const int a = tid & 31, part = tid >> 5;
        float tot = 0.f;
        if (a < q)
            for (int t = part; t < ntiles; t += 8) tot += gh_part[((int64_t)i * ntiles + t) * S + a];
        __shared__ float s_p[8][32];
        s_p[part][a] = tot;
        __syncthreads();
        if (tid < q) {
            float v = 0.f;
            for (int p = 0; p < 8; p++) v += s_p[p][tid];
            gh[i * q + tid] = v;
        }
        return;
    }
    if (fx != nullptr) {
        double acc = 0.0;
        for (int64_t e = tid; e < (int64_t)L * ntiles; e += blockDim.x) acc += fx_part[e];
        s_red[tid] = acc;
        __syncthreads();
        for (int o = 128; o > 0; o >>= 1) {
            if (tid < o) s_red[tid] += s_red[tid + o];
            __syncthreads();
        }
        if (tid == 0) fx[0] = s_red[0];
    }
}

int plm_finalize(const PlmGeom &g, const float *d_G, const float *d_gh_part, const double *d_fx_part,
                 float *d_gh, float *d_gJ, double *d_fx, float scale_pair, cudaStream_t st)
{
    dim3 grid((unsigned)g.L, (unsigned)g.L);
    finalize_pairs_kernel<<<grid, 128, 0, st>>>(d_G, d_gJ, g.L, g.Lp, g.q, g.QB, g.S, scale_pair);
    EVC_KERNEL_CHECK();
    finalize_fields_kernel<<<g.L + 1, 256, 0, st>>>(d_gh_part, d_fx_part, d_gh, d_fx, g.L, g.q, g.S, g.ntiles_f);
    EVC_KERNEL_CHECK();
    return 0;
}

int plm_finalize_fields_n(const PlmGeom &g, const float *d_gh_part, const double *d_fx_part, float *d_gh,
                          double *d_fx, int ntiles, cudaStream_t st)
{
    finalize_fields_kernel<<<g.L + 1, 256, 0, st>>>(d_gh_part, d_fx_part, d_gh, d_fx, g.L, g.q, g.S, ntiles);
    EVC_KERNEL_CHECK();
    return 0;
}

int plm_finalize_fields(const PlmGeom &g, const float *d_gh_part, const double *d_fx_part, float *d_gh,
                        double *d_fx, cudaStream_t st)
{
    finalize_fields_kernel<<<g.L + 1, 256, 0, st>>>(d_gh_part, d_fx_part, d_gh, d_fx, g.L, g.q, g.S, g.ntiles_f);
    EVC_KERNEL_CHECK();
    return 0;
}

}  // namespace evc
