// Hot path (b): O(N^2 L) pairwise-Hamming sequence reweighting on sm_90a.
//
// Replaces plmc's reweighting pass and the in-tree numba twin
// evcouplings/align/alignment.py:1192-1233 (num_cluster_members): for every
// sequence s, count the sequences t (self included) with at least
// `min_identical` identical positions (gap == gap is an identity).
//
// Data layout: the uint8 code matrix (codes < 32) is transposed once into five
// bit-planes  planes[p][w][n]  (bit k of word w = bit p of the code at site
// 32w+k, n fastest so a warp reads 128 contiguous bytes).  Two sequences agree
// at a site iff all five plane bits agree, so one 32-site word of a pair costs
// 5 LOP3 + 1 POPC + 1 IADD -- ~6.6x fewer instructions than byte compares and
// integer-exact.  Padded sites (32*W - L) are zero in every sequence and are
// accounted for by raising the threshold.
//
// Tiling: 128 x 128 pair tiles over the upper triangle (each unordered pair
// visited once; a tile credits both its rows and its columns), 256 threads,
// 8x8 pair counters per thread in registers, plane words staged in shared
// memory 16 words (512 sites) at a time.  The plane buffer (N * 5 * W * 4 bytes; 40 MB at
// N=200k, L=300) is L2-resident, so the kernel is bound by the integer pipes.
#include <stdlib.h>

#include <algorithm>

#include <map>
#include <mutex>
#include <utility>

#include "common.cuh"
#include "internal.h"

namespace evc {

constexpr int HP = 5;        // bit planes (codes < 32)
constexpr int HT = 128;      // pair-tile edge
constexpr int HWC = 16;      // words staged per step (80 KB of dynamic shared memory => 2 CTAs / SM)

__global__ void hamming_pack_kernel(const uint8_t *__restrict__ codes, int64_t N, int L, int W,
                                    uint32_t *__restrict__ planes)
{
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int w = blockIdx.y;
    if (n >= N) return;
    uint32_t pl[HP] = {0, 0, 0, 0, 0};
    const uint8_t *row = codes + n * L;
    const int k0 = w * 32;
#pragma unroll 4
    for (int k = 0; k < 32; k++) {
        const int site = k0 + k;
        const uint32_t c = site < L ? row[site] : 0u;
#pragma unroll
        for (int p = 0; p < HP; p++) pl[p] |= ((c >> p) & 1u) << k;
    }
#pragma unroll
    for (int p = 0; p < HP; p++) planes[((int64_t)p * W + w) * N + n] = pl[p];
}

__device__ __forceinline__ void tile_from_index(int64_t idx, int64_t T, int64_t &R, int64_t &C)
{
    // idx enumerates (R, C >= R) row-major: offset(R) = R*T - R(R-1)/2
    double t = (double)(2 * T + 1);
    int64_t r = (int64_t)floor((t - sqrt(t * t - 8.0 * (double)idx)) * 0.5);
    if (r < 0) r = 0;
    if (r > T - 1) r = T - 1;
    while (r > 0 && r * T - r * (r - 1) / 2 > idx) r--;
    while ((r + 1) * T - (r + 1) * r / 2 <= idx) r++;
    R = r;
    C = r + (idx - (r * T - r * (r - 1) / 2));
}

// Column owned by counter c of thread tx: {4 tx .. 4 tx + 3} and {64 + 4 tx .. 64 + 4 tx + 3}.  A quarter warp then
// reads 8 x 16 contiguous bytes of s_col per 128-bit load (conflict-free); the round-1 mapping 8 tx + c put
// threads tx and tx + 4 on the same banks (2-way conflicts).
__device__ __forceinline__ int hcol(int tx, int c) { return (c < 4) ? tx * 4 + c : 64 + tx * 4 + (c - 4); }

// FILTER = false: full comparison, neighbour counts credited directly (with exact early termination).
// FILTER = true : phase 1 of the two-phase scheme -- only the first W1 plane words are compared; a pair whose
//                 identities so far plus everything it could still gain reach the threshold is appended to a
//                 candidate list (row, col | credit-both flag) for exact verification by hamming_verify_kernel.
// MULT = true   : rows are distinct rows with multiplicities mult[]: a neighbour pair credits mult[col] to its row and
//                 mult[row] to its column instead of 1 (the filter never credits, so it has no MULT version).
template <bool FILTER, bool MULT = false>
__global__ void __launch_bounds__(256, 2)
hamming_tile_kernel(const uint32_t *__restrict__ planes, int64_t N, int W, int thr,
                    int64_t tile_begin, int64_t T, int *__restrict__ counts, int W1,
                    uint2 *__restrict__ cand, unsigned long long *__restrict__ cand_count,
                    unsigned long long cand_cap, const int *__restrict__ mult = nullptr)
{
    extern __shared__ __align__(16) uint32_t s_dyn[];
    uint32_t (*s_row)[HP][HT] = reinterpret_cast<uint32_t (*)[HP][HT]>(s_dyn);
    uint32_t (*s_col)[HP][HT] = reinterpret_cast<uint32_t (*)[HP][HT]>(s_dyn + HWC * HP * HT);
    __shared__ int s_rsum[HT];
    __shared__ int s_csum[HT];

    int64_t R, C;
    tile_from_index(tile_begin + blockIdx.x, T, R, C);
    const int64_t row0 = R * HT, col0 = C * HT;
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;

    int cnt[8][8];
#pragma unroll
    for (int r = 0; r < 8; r++)
#pragma unroll
        for (int c = 0; c < 8; c++) cnt[r][c] = 0;
    if (tid < HT) { s_rsum[tid] = 0; s_csum[tid] = 0; }

    // Exact early termination at warp granularity: after word w a pair can still gain at most 32 * (W - 1 - w)
    // identities; a warp (16 x 128 pairs) whose pairs can no longer reach the threshold stops comparing (it only
    // keeps arriving at the staging barriers), and the tile ends when all of its warps are done.
    bool wdead = false;
    const int Wrun = FILTER ? W1 : W;
    for (int w0 = 0; w0 < Wrun; w0 += HWC) {
        const int nw = min(HWC, Wrun - w0);
        if (!__syncthreads_or(!wdead)) break;
        // stage nw words x 5 planes x 128 sequences for both sides
        for (int e = tid; e < HWC * HP * HT; e += 256) {
            const int s = e & (HT - 1);
            const int p = (e / HT) % HP;
            const int ww = e / (HT * HP);
            uint32_t vr = 0, vc = 0;
            if (ww < nw) {
                const int64_t base = ((int64_t)p * W + (w0 + ww)) * N;
                if (row0 + s < N) vr = planes[base + row0 + s];
                if (col0 + s < N) vc = planes[base + col0 + s];
            }
            s_row[ww][p][s] = vr;
            s_col[ww][p][s] = vc;
        }
        __syncthreads();
        for (int ww = 0; ww < nw && !wdead; ww++) {
            uint32_t a[HP][8], b[HP][8];
#pragma unroll
            for (int p = 0; p < HP; p++) {
                const uint4 a0 = *reinterpret_cast<const uint4 *>(&s_row[ww][p][ty * 8]);
                const uint4 a1 = *reinterpret_cast<const uint4 *>(&s_row[ww][p][ty * 8 + 4]);
                const uint4 b0 = *reinterpret_cast<const uint4 *>(&s_col[ww][p][tx * 4]);
                const uint4 b1 = *reinterpret_cast<const uint4 *>(&s_col[ww][p][64 + tx * 4]);
                a[p][0] = a0.x; a[p][1] = a0.y; a[p][2] = a0.z; a[p][3] = a0.w;
                a[p][4] = a1.x; a[p][5] = a1.y; a[p][6] = a1.z; a[p][7] = a1.w;
                b[p][0] = b0.x; b[p][1] = b0.y; b[p][2] = b0.z; b[p][3] = b0.w;
                b[p][4] = b1.x; b[p][5] = b1.y; b[p][6] = b1.z; b[p][7] = b1.w;
            }
#pragma unroll
            for (int r = 0; r < 8; r++)
#pragma unroll
                for (int c = 0; c < 8; c++) {
                    uint32_t d = a[0][r] ^ b[0][c];
#pragma unroll
                    for (int p = 1; p < HP; p++) d |= a[p][r] ^ b[p][c];
                    cnt[r][c] += __popc(~d);
                }
            const int wdone = w0 + ww;
            if (!FILTER && W1 >= 0 && wdone >= 1 && wdone + 1 < W) {      // W1 < 0: early termination disabled (bench hook)
                const int need = thr - 32 * (W - 1 - wdone);
                int alive = 0;
#pragma unroll
                for (int r = 0; r < 8; r++)
#pragma unroll
                    for (int c = 0; c < 8; c++) alive |= (cnt[r][c] >= need);
                if (!__any_sync(0xffffffffu, alive)) wdead = true;
            }
        }
    }

    const bool diag = (R == C);
    if (FILTER) {
        // candidates: identities in the first W1 words + the 32 * (W - W1) still possible >= threshold.
        // One atomic per warp: lane-local counts -> warp prefix sum -> the warp reserves a contiguous range.
        const int need = thr - 32 * (W - W1);
        int mine = 0;
#pragma unroll
        for (int r = 0; r < 8; r++)
#pragma unroll
            for (int c = 0; c < 8; c++)
                mine += (row0 + ty * 8 + r < N && col0 + hcol(tx, c) < N && cnt[r][c] >= need) ? 1 : 0;
        const int lane = tid & 31;
        int incl = mine;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += u;
        }
        const int total = __shfl_sync(0xffffffffu, incl, 31);
        if (total == 0) return;
        unsigned long long base = 0;
        if (lane == 0) base = atomicAdd(cand_count, (unsigned long long)total);
        base = __shfl_sync(0xffffffffu, base, 0);
        unsigned long long slot = base + (unsigned long long)(incl - mine);
#pragma unroll
        for (int r = 0; r < 8; r++)
#pragma unroll
            for (int c = 0; c < 8; c++) {
                const int64_t gr = row0 + ty * 8 + r, gc = col0 + hcol(tx, c);
                if (gr < N && gc < N && cnt[r][c] >= need) {
                    if (slot < cand_cap)
                        cand[slot] = make_uint2((unsigned)gr, (unsigned)gc | (diag ? 0u : 0x80000000u));
                    slot++;
                }
            }
        return;
    }
    // threshold -> neighbour flags; credit rows (always) and columns (off-diagonal tiles)
    int rs[8], cs[8];
    int mr[8], mc[8];                                 // multiplicities of this thread's rows / columns (MULT)
#pragma unroll
    for (int r = 0; r < 8; r++) rs[r] = 0;
#pragma unroll
    for (int c = 0; c < 8; c++) cs[c] = 0;
    if (MULT) {
#pragma unroll
        for (int r = 0; r < 8; r++) mr[r] = row0 + ty * 8 + r < N ? mult[row0 + ty * 8 + r] : 0;
#pragma unroll
        for (int c = 0; c < 8; c++) mc[c] = col0 + hcol(tx, c) < N ? mult[col0 + hcol(tx, c)] : 0;
    }
#pragma unroll
    for (int r = 0; r < 8; r++)
#pragma unroll
        for (int c = 0; c < 8; c++) {
            const bool ok = (row0 + ty * 8 + r < N) && (col0 + hcol(tx, c) < N);
            const int f = (ok && cnt[r][c] >= thr) ? 1 : 0;
            if (MULT) {
                rs[r] += f * mc[c];
                cs[c] += f * mr[r];
            } else {
                rs[r] += f;
                cs[c] += f;
            }
        }
#pragma unroll
    for (int r = 0; r < 8; r++)
        if (rs[r]) atomicAdd(&s_rsum[ty * 8 + r], rs[r]);
    if (!diag) {
#pragma unroll
        for (int c = 0; c < 8; c++)
            if (cs[c]) atomicAdd(&s_csum[hcol(tx, c)], cs[c]);
    }
    __syncthreads();
    if (tid < HT) {
        if (row0 + tid < N && s_rsum[tid]) atomicAdd(&counts[row0 + tid], s_rsum[tid]);
    } else if (tid < 2 * HT && !diag) {
        const int c = tid - HT;
        if (col0 + c < N && s_csum[c]) atomicAdd(&counts[col0 + c], s_csum[c]);
    }
}

// phase 2: exact identity count of every candidate pair over all W words (thread = candidate); MULT credits
// multiplicities as the tile kernel does
template <bool MULT = false>
__global__ void hamming_verify_kernel(const uint32_t *__restrict__ planes, int64_t N, int W, int thr,
                                      const uint2 *__restrict__ cand, unsigned long long ncand,
                                      int *__restrict__ counts, const int *__restrict__ mult = nullptr)
{
    const unsigned long long k = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= ncand) return;
    const uint2 pr = cand[k];
    const int64_t r = pr.x, c = pr.y & 0x7fffffffu;
    const bool both = (pr.y & 0x80000000u) != 0;
    int cnt = 0;
    for (int w = 0; w < W; w++) {
        uint32_t d = 0;
#pragma unroll
        for (int p = 0; p < HP; p++) {
            const int64_t base = ((int64_t)p * W + w) * N;
            d |= planes[base + r] ^ planes[base + c];
        }
        cnt += __popc(~d);
    }
    if (cnt >= thr) {
        atomicAdd(&counts[r], MULT ? mult[c] : 1);
        if (both) atomicAdd(&counts[c], MULT ? mult[r] : 1);
    }
}

// test / bench hooks, read once per process (tests drive them from subprocesses)
static long long env_once(const char *name, long long *cache)
{
    if (*cache == -2) {
        const char *e = getenv(name);
        *cache = e ? atoll(e) : -1;
    }
    return *cache;
}
static long long g_env_cap = -2, g_env_single = -2, g_env_noprune = -2;

struct HammingScratch {
    uint2 *cand = nullptr;
    unsigned long long *count = nullptr;
    unsigned long long cap = 0;
};
// candidate buffers per (device, stream): concurrent reweighting passes on different streams do not share one (ADVICE r1)
static std::mutex g_hs_mutex;
static std::map<std::pair<int, cudaStream_t>, HammingScratch> g_hs;

static int hamming_scratch(unsigned long long want, cudaStream_t st, HammingScratch **out)
{
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { set_error("hamming: bad device"); return 1; }
    std::lock_guard<std::mutex> lock(g_hs_mutex);
    HammingScratch &h = g_hs[std::make_pair(dev, st)];
    if (!h.count && cudaMalloc(&h.count, sizeof(unsigned long long)) != cudaSuccess) {
        h.count = nullptr;
        set_error("hamming: scratch allocation failed");
        return 1;
    }
    if (h.cap != want && (h.cap < want || env_once("EVC_HAMMING_CAND_CAP", &g_env_cap) > 0)) {
        cudaFree(h.cand);
        h.cand = nullptr;
        h.cap = 0;
        if (cudaMalloc(&h.cand, want * sizeof(uint2)) != cudaSuccess) {
            cudaGetLastError();
            set_error("hamming: candidate buffer allocation failed");
            return 1;
        }
        h.cap = want;
    }
    *out = &h;
    return 0;
}

// f3: identities of every sequence to one target sequence (reference twin evcouplings/align/alignment.py:1156-1189):
// warp = sequence, lanes stride over the sites (coalesced 32-byte segments), shuffle reduction.  HBM-streaming.
__global__ void identities_to_seq_kernel(const uint8_t *__restrict__ codes, const uint8_t *__restrict__ seq, int64_t N,
                                         int L, int *__restrict__ out)
{
    const int64_t n = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (n >= N) return;
    const uint8_t *row = codes + n * L;
    int acc = 0;
    for (int j = lane; j < L; j += 32) acc += (row[j] == seq[j]) ? 1 : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) out[n] = acc;
}

int identities_to_seq(const uint8_t *d_codes, const uint8_t *d_seq, int64_t N, int L, int *d_out, cudaStream_t st)
{
    if (N <= 0 || L <= 0) { set_error("identities_to_seq: empty alignment"); return 1; }
    identities_to_seq_kernel<<<(unsigned)ceil_div(N, 8), 256, 0, st>>>(d_codes, d_seq, N, L, d_out);
    EVC_KERNEL_CHECK();
    return 0;
}

int64_t hamming_plane_words(int64_t N, int L) { return (int64_t)HP * ceil_div(L, 32) * N; }

int64_t hamming_num_tiles(int64_t N)
{
    const int64_t T = ceil_div(N, HT);
    return T * (T + 1) / 2;
}

int hamming_pack(const uint8_t *d_codes, int64_t N, int L, uint32_t *d_planes, cudaStream_t st)
{
    if (N <= 0 || L <= 0) { set_error("hamming_pack: empty alignment"); return 1; }
    const int W = (int)ceil_div(L, 32);
    dim3 grid((unsigned)ceil_div(N, 256), (unsigned)W);
    hamming_pack_kernel<<<grid, 256, 0, st>>>(d_codes, N, L, W, d_planes);
    EVC_KERNEL_CHECK();
    return 0;
}

int hamming_count_tiles(const uint32_t *d_planes, const int *d_mult, int64_t N, int L, int min_identical,
                        int64_t tile_begin, int64_t tile_end, int *d_counts, cudaStream_t st)
{
    const int W = (int)ceil_div(L, 32);
    const int64_t T = ceil_div(N, HT);
    if (tile_begin < 0 || tile_end > T * (T + 1) / 2 || tile_begin > tile_end) {
        set_error("hamming_count_tiles: tile range out of bounds");
        return 1;
    }
    const size_t smem = (size_t)2 * HWC * HP * HT * sizeof(uint32_t);
    EVC_CUDA(cudaFuncSetAttribute(hamming_tile_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    EVC_CUDA(cudaFuncSetAttribute(hamming_tile_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    if (d_mult)
        EVC_CUDA(cudaFuncSetAttribute(hamming_tile_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)smem));
    const int thr = min_identical + (W * 32 - L);   // padded sites always "agree"
    const int64_t ntile = tile_end - tile_begin;
    if (ntile == 0) return 0;

    // Two-phase scheme for long alignments: filter on the first ~30 % of the words, verify the survivors.
    // The filter only pays when it can reject: the identities still obtainable after W1 words, 32 * (W - W1),
    // must be well below the threshold.  Falls back to the single-phase kernel if the candidate list overflows.
    const int W1 = (W * 3 + 9) / 10;
    const bool no_prune = env_once("EVC_HAMMING_NO_PRUNE", &g_env_noprune) > 0;    // bench: un-pruned reference time
    const bool two_phase = W >= 6 && (thr - 32 * (W - W1)) >= 8 && !no_prune &&
                           env_once("EVC_HAMMING_SINGLE_PHASE", &g_env_single) <= 0;
    if (two_phase) {
        HammingScratch *hs = nullptr;
        unsigned long long want = (unsigned long long)std::min<int64_t>((int64_t)1 << 27, std::max<int64_t>(N * 512, 1 << 20));
        if (env_once("EVC_HAMMING_CAND_CAP", &g_env_cap) > 0) want = (unsigned long long)g_env_cap;   // tests
        if (hamming_scratch(want, st, &hs) == 0) {
            EVC_CUDA(cudaMemsetAsync(hs->count, 0, sizeof(unsigned long long), st));
            int64_t done = tile_begin;
            while (done < tile_end) {
                const int64_t nblk = std::min<int64_t>(tile_end - done, (int64_t)1 << 30);
                hamming_tile_kernel<true><<<(unsigned)nblk, 256, smem, st>>>(d_planes, N, W, thr, done, T, d_counts, W1,
                                                                             hs->cand, hs->count, want);
                EVC_KERNEL_CHECK();
                done += nblk;
            }
            unsigned long long ncand = 0;
            EVC_CUDA(cudaMemcpyAsync(&ncand, hs->count, sizeof(ncand), cudaMemcpyDeviceToHost, st));
            EVC_CUDA(cudaStreamSynchronize(st));
            if (ncand <= want) {
                if (ncand > 0) {
                    const unsigned nb = (unsigned)((ncand + 255) / 256);
                    if (d_mult)
                        hamming_verify_kernel<true><<<nb, 256, 0, st>>>(d_planes, N, W, thr, hs->cand, ncand, d_counts,
                                                                        d_mult);
                    else
                        hamming_verify_kernel<<<nb, 256, 0, st>>>(d_planes, N, W, thr, hs->cand, ncand, d_counts);
                    EVC_KERNEL_CHECK();
                }
                return 0;
            }
            // overflow: nothing has been credited yet (the filter never touches counts) -> single phase below
        }
    }
    int64_t done = tile_begin;
    while (done < tile_end) {                        // grid.x limit 2^31-1
        const int64_t nblk = std::min<int64_t>(tile_end - done, (int64_t)1 << 30);
        if (d_mult)
            hamming_tile_kernel<false, true><<<(unsigned)nblk, 256, smem, st>>>(
                d_planes, N, W, thr, done, T, d_counts, no_prune ? -1 : W, nullptr, nullptr, 0, d_mult);
        else
            hamming_tile_kernel<false><<<(unsigned)nblk, 256, smem, st>>>(d_planes, N, W, thr, done, T, d_counts,
                                                                          no_prune ? -1 : W, nullptr, nullptr, 0);
        EVC_KERNEL_CHECK();
        done += nblk;
    }
    return 0;
}

}  // namespace evc
