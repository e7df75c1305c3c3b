// Distinct rows of the code matrix (evc_msa_unique): which rows of an N x L uint8 alignment are exact repeats of an
// earlier row.  The reweighting pass, the pair counts and every objective evaluation are sums over rows whose terms
// depend only on the row's codes and its weight, so they can run once per distinct row with the row's multiplicity.
//
// Exact and deterministic:
//   1. a 64-bit hash per row (warp per row; a position-mixed sum of splitmix64 finalizers, so the lanes' partial
//      sums combine in any order to the same value);
//   2. a stable LSD radix sort of (hash, row) pairs (CUB): rows of one hash group stay in ascending row order;
//   3. every row is compared byte for byte with the rows before it in its hash group; the first equal one (the
//      group's earliest copy of that row, since the group is in row order) is its representative.  A hash collision
//      only makes a group longer: rows merge only if all L codes are equal;
//   4. an exclusive scan over the "is its own representative" flags, in row order, numbers the distinct rows in
//      ascending order of their first occurrence; multiplicities are integer atomics.
// Scratch: 40 bytes per row plus CUB's temporary storage, allocated stream-ordered on the caller's stream.
#include <stdlib.h>

#include <algorithm>

#include <cub/cub.cuh>

#include "common.cuh"
#include "internal.h"

namespace evc {

__global__ void unique_hash_kernel(const uint8_t *__restrict__ codes, int64_t N, int L, uint64_t mask,
                                   uint64_t *__restrict__ keys, int *__restrict__ rows)
{
    const int64_t n = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (n >= N) return;
    const uint8_t *row = codes + n * L;
    uint64_t acc = 0;
    for (int j = lane; j < L; j += 32) acc += splitmix64_mix((uint64_t)(j + 1) * GOLDEN_GAMMA ^ row[j]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) {
        keys[n] = acc & mask;
        rows[n] = (int)n;
    }
}

// start of each sorted position's hash group (inclusive max-scan of these gives it)
__global__ void unique_group_head_kernel(const uint64_t *__restrict__ keys, int64_t N, int *__restrict__ head)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    head[i] = (i == 0 || keys[i] != keys[i - 1]) ? (int)i : 0;
}

// representative of the row at sorted position i: the first row of its hash group with the same L codes
__global__ void unique_rep_kernel(const uint8_t *__restrict__ codes, int64_t N, int L, const int *__restrict__ rows,
                                  const int *__restrict__ group, int *__restrict__ rep, int *__restrict__ is_first)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const int r = rows[i];
    const uint8_t *a = codes + (int64_t)r * L;
    int found = r;
    for (int64_t j = group[i]; j < i; j++) {
        const int c = rows[j];
        const uint8_t *b = codes + (int64_t)c * L;
        int k = 0;
        while (k < L && a[k] == b[k]) k++;
        if (k == L) {
            found = c;
            break;
        }
    }
    rep[r] = found;
    is_first[r] = found == r ? 1 : 0;
}

__global__ void unique_finish_kernel(int64_t N, const int *__restrict__ rep, const int *__restrict__ is_first,
                                     const int *__restrict__ pos, int *__restrict__ first, int *__restrict__ inverse,
                                     int *__restrict__ mult, int *__restrict__ d_U)
{
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= N) return;
    if (is_first[r]) first[pos[r]] = (int)r;
    const int u = pos[rep[r]];
    inverse[r] = u;
    atomicAdd(&mult[u], 1);
    if (r == N - 1) *d_U = pos[r] + is_first[r];
}

struct MaxOp {
    __device__ __forceinline__ int operator()(int a, int b) const { return a > b ? a : b; }
};

int msa_unique(const uint8_t *d_codes, int64_t N, int L, int *d_first, int *d_inverse, int *d_mult, int64_t *U_out,
               cudaStream_t st)
{
    if (N <= 0 || L <= 0) { set_error("evc_msa_unique: empty alignment"); return 1; }
    if (N >= ((int64_t)1 << 31)) { set_error("evc_msa_unique: N must be below 2^31 (int32 row indices)"); return 1; }
    // test hook: keep only the low EVC_UNIQUE_HASH_BITS bits of the hash, so that distinct rows collide
    int bits = 64;
    if (const char *e = getenv("EVC_UNIQUE_HASH_BITS")) bits = std::max(1, std::min(64, atoi(e)));
    const uint64_t mask = bits == 64 ? ~0ull : ((1ull << bits) - 1);
    const int n = (int)N;

    size_t sort_bytes = 0, scan_bytes = 0, sum_bytes = 0;
    EVC_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const uint64_t *)nullptr, (uint64_t *)nullptr,
                                             (const int *)nullptr, (int *)nullptr, n, 0, bits, st));
    EVC_CUDA(cub::DeviceScan::InclusiveScan(nullptr, scan_bytes, (const int *)nullptr, (int *)nullptr, MaxOp(), n, st));
    EVC_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, sum_bytes, (const int *)nullptr, (int *)nullptr, n, st));
    const size_t temp_bytes = round_up((int64_t)std::max(sort_bytes, std::max(scan_bytes, sum_bytes)), 256);
    const size_t key_bytes = round_up(N * 8, 256), int_bytes = round_up(N * 4, 256);
    const size_t total = 2 * key_bytes + 6 * int_bytes + 256 + temp_bytes;
    char *buf = nullptr;
    if (cudaMallocAsync(&buf, total, st) != cudaSuccess) {
        cudaGetLastError();
        set_error("evc_msa_unique: scratch allocation failed");
        return 1;
    }
    uint64_t *keys = (uint64_t *)buf, *keys_s = (uint64_t *)(buf + key_bytes);
    int *ib = (int *)(buf + 2 * key_bytes);
    const size_t iw = int_bytes / 4;
    int *rows = ib, *rows_s = ib + iw, *group = ib + 2 * iw, *rep = ib + 3 * iw, *is_first = ib + 4 * iw,
        *pos = ib + 5 * iw;
    int *d_U = ib + 6 * iw;
    void *temp = buf + 2 * key_bytes + 6 * int_bytes + 256;

    // every step runs only while the previous ones succeeded; the scratch is freed on every path
    cudaError_t e = cudaSuccess;
    const unsigned blocks = (unsigned)ceil_div(N, 256);
    size_t tb = temp_bytes;
    unique_hash_kernel<<<(unsigned)ceil_div(N, 8), 256, 0, st>>>(d_codes, N, L, mask, keys, rows);
    e = cudaGetLastError();
    if (e == cudaSuccess) e = cub::DeviceRadixSort::SortPairs(temp, tb, keys, keys_s, rows, rows_s, n, 0, bits, st);
    if (e == cudaSuccess) {
        unique_group_head_kernel<<<blocks, 256, 0, st>>>(keys_s, N, group);
        e = cudaGetLastError();
    }
    tb = temp_bytes;
    if (e == cudaSuccess) e = cub::DeviceScan::InclusiveScan(temp, tb, group, group, MaxOp(), n, st);
    if (e == cudaSuccess) {
        unique_rep_kernel<<<blocks, 256, 0, st>>>(d_codes, N, L, rows_s, group, rep, is_first);
        e = cudaGetLastError();
    }
    tb = temp_bytes;
    if (e == cudaSuccess) e = cub::DeviceScan::ExclusiveSum(temp, tb, is_first, pos, n, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_mult, 0, (size_t)N * sizeof(int), st);
    if (e == cudaSuccess) {
        unique_finish_kernel<<<blocks, 256, 0, st>>>(N, rep, is_first, pos, d_first, d_inverse, d_mult, d_U);
        e = cudaGetLastError();
    }
    int U = 0;
    if (e == cudaSuccess) e = cudaMemcpyAsync(&U, d_U, sizeof(int), cudaMemcpyDeviceToHost, st);
    cudaFreeAsync(buf, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) {
        set_error(std::string("evc_msa_unique: ") + cudaGetErrorString(e));
        return 1;
    }
    *U_out = U;
    return 0;
}

}  // namespace evc
