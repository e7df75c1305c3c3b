// Gibbs sampler of a fitted Potts model (evc_sampler_*; the chain's contract is in include/evcplm.h).
//
// One warp per chain.  The chain's field row Z (L*q fp32) and its codes live in shared memory for the whole call;
// a CTA holds as many chains as its shared memory allows (SAMPLE_SMEM_MAX) up to SAMPLE_MAX_WARPS.  Per site the
// lanes a < q hold beta * Z_i(a), the warp takes the max and the inclusive prefix sum of exp(v - max) by shuffles
// and draws; only when s_i changes does it stream the two rows U[(i,b), :] and U[(i,a), :] (8 L q bytes) and add
// their difference into Z.  Chains never wait for each other: there is no barrier per site.
//
// U is the full symmetric coupling matrix, (L q) x (L q) fp32, row (i,a) holding J_ij(a, .) for every j and zero
// diagonal blocks, built once per handle from x.  Its symmetry makes the refresh of Z from s a sum of whole rows:
// Z(i,a) = h_i(a) + sum_j U[(j, s_j), (i,a)], j ascending, coalesced along (i,a).
//
// Z persists in device memory between calls, so a run split over calls is bit-identical to one call: the refresh
// happens at global sweep indices t % EVC_SAMPLER_REFRESH == 0, never at a call boundary.  The one exception is
// evc_sampler_set_model, which loads new parameters: the sweep after it refreshes too (refresh_first).
//
// evc_sampler_anneal runs the same kernel instantiated with ANNEAL: couplings scaled by a per-sweep beta, and a
// per-chain log importance weight read off the field row Z before each sweep (annealed importance sampling).
#include "../../include/evcplm.h"

#include <math.h>
#include <stdlib.h>

#include <algorithm>
#include <new>
#include <string>
#include <vector>

#include "common.cuh"

namespace evc {

constexpr int SAMPLE_SMEM_MAX = 227 * 1024;     // opt-in shared memory of one sm_90 CTA
constexpr int SAMPLE_MAX_WARPS = 16;

static int64_t sample_row_bytes(int L, int q) { return round_up((int64_t)L * q * 4 + L, 16); }

__host__ __device__ __forceinline__ uint64_t sample_chain_key(uint64_t seed, uint64_t c)
{
    return splitmix64_mix(seed ^ splitmix64_mix((c + 1ull) * GOLDEN_GAMMA));
}

// the top 24 bits of the counter's hash: u = (draw + 0.5) * 2^-24
__device__ __forceinline__ uint32_t sample_draw24(uint64_t key, int64_t t, int L, int i)
{
    const uint64_t k = (uint64_t)t * (uint64_t)L + (uint64_t)i + 1ull;
    return (uint32_t)(splitmix64_mix(key + k * GOLDEN_GAMMA) >> 40);
}

__global__ void sample_build_u_kernel(const float *__restrict__ J, int L, int q, float *__restrict__ U)
{
    const int Lq = L * q;
    const int r = blockIdx.y;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= Lq) return;
    const int i = r / q, a = r - i * q, j = e / q, b = e - j * q;
    float v = 0.f;
    if (i < j) v = J[((int64_t)i * L - (int64_t)i * (i + 1) / 2 + (j - i - 1)) * q * q + a * q + b];
    else if (j < i) v = J[((int64_t)j * L - (int64_t)j * (j + 1) / 2 + (i - j - 1)) * q * q + b * q + a];
    U[(int64_t)r * Lq + e] = v;
}

// uniform start (t = -1): s_i = floor(u q), computed exactly as ((2 draw + 1) q) >> 25
__global__ void sample_uniform_start_kernel(uint8_t *__restrict__ codes, int64_t n_chains, int64_t chain_offset,
                                            uint64_t seed, int L, int q)
{
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_chains * L) return;
    const int64_t c = e / L;
    const int i = (int)(e - c * L);
    const uint64_t d = sample_draw24(sample_chain_key(seed, (uint64_t)(chain_offset + c)), -1, L, i);
    codes[e] = (uint8_t)(((2ull * d + 1ull) * (uint64_t)q) >> 25);
}

// v = h + beta (Z - h), each operation rounded on its own: no contraction, so the float64 restatement can repeat it
__device__ __forceinline__ float annealed_logit(float h, float z, float beta)
{
    return __fadd_rn(h, __fmul_rn(beta, __fsub_rn(z, h)));
}

// H = sum_i h_i(s_i) + 1/2 sum_i (Z_i(s_i) - h_i(s_i)) over n sites in double, every lane of the warp taking the sites
// k = lane, lane + 32, ... and the butterfly adding the lanes' sums: each lane ends with the same value (each step adds
// the same two values in either order).  The order is that of the ANNEAL path's H_J.
__device__ __forceinline__ double chain_energy(const float *z, const float *h, const uint8_t *s, int n, int q, int lane)
{
    double eh = 0.0, ej = 0.0;
    for (int k = lane; k < n; k += 32) {
        const int r = k * q + s[k];
        const double hr = (double)h[r];
        eh = __dadd_rn(eh, hr);
        ej = __dadd_rn(ej, __dsub_rn((double)z[r], hr));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        eh = __dadd_rn(eh, __shfl_xor_sync(0xffffffffu, eh, o));
        ej = __dadd_rn(ej, __shfl_xor_sync(0xffffffffu, ej, o));
    }
    return __dadd_rn(eh, __dmul_rn(0.5, ej));
}

// ANNEAL (evc_sampler_anneal): sweep t0 + k runs at betas[k + 1] and draws from v_a = h_i(a) + beta (Z_i(a) - h_i(a));
// before it, once any refresh due has run, the chain's log weight gains (betas[k + 1] - betas[k]) H_J(s) with
// H_J = 1/2 sum_i (Z_i(s_i) - h_i(s_i)) in double.  The plain instantiation ignores betas and logw.
//
// TEMPER (evc_sampler_temper): the plain sweep at the chain's own beta, betas[c] (the rung it holds, read once per
// call); when logw is not null the call ends on a swap round and logw[c] receives the chain's energy (chain_energy).
//
// RECORD (evc_sampler_record_best; plain and TEMPER only): after every sweep t the chain forms H with chain_energy and,
// if H > best_energy[c] (strictly, so a NaN H never counts), stores H, its codes and t.  The record only reads z and s,
// so the chain itself is that of the instantiation without it.
template <bool ANNEAL, bool TEMPER = false, bool RECORD = false>
__global__ void __launch_bounds__(32 * SAMPLE_MAX_WARPS)
sample_gibbs_kernel(const float *__restrict__ U, const float *__restrict__ h, float *__restrict__ Zg,
                    uint8_t *__restrict__ codes, unsigned long long *__restrict__ changes, int L, int q,
                    int64_t n_chains, int64_t chain_offset, uint64_t seed, int64_t t0, int sweeps, float beta,
                    int row_bytes, bool refresh_first, const float *__restrict__ betas, double *__restrict__ logw,
                    double *__restrict__ best_energy, uint8_t *__restrict__ best_codes,
                    int64_t *__restrict__ best_sweep)
{
    static_assert(!(ANNEAL && RECORD), "annealing does not record");
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t c = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
    if (c >= n_chains) return;                  // the whole warp: no CTA barrier below
    if constexpr (TEMPER) beta = betas[c];
    const int Lq = L * q;
    float *z = reinterpret_cast<float *>(smem_raw + (size_t)warp * row_bytes);
    uint8_t *s = reinterpret_cast<uint8_t *>(z + Lq);
    float *zc = Zg + c * Lq;
    uint8_t *sc = codes + c * L;
    for (int k = lane; k < L; k += 32) s[k] = sc[k];
    if (t0 % EVC_SAMPLER_REFRESH != 0 && !refresh_first)
        for (int e = lane; e < Lq; e += 32) z[e] = zc[e];
    __syncwarp();
    const uint64_t key = sample_chain_key(seed, (uint64_t)(chain_offset + c));
    unsigned long long changed = 0;
    double w = 0.0;
    if constexpr (ANNEAL) w = logw[c];
    double best = 0.0;
    int64_t best_t = -1;                        // the sweep of this call's last new record, -1: none
    if constexpr (RECORD) best = best_energy[c];
    for (int64_t t = t0; t < t0 + sweeps; t++) {
        if (t % EVC_SAMPLER_REFRESH == 0 || (refresh_first && t == t0)) {
            for (int e = lane; e < Lq; e += 32) {
                float acc = h[e];
                for (int j = 0; j < L; j++) acc += U[(int64_t)(j * q + s[j]) * Lq + e];
                z[e] = acc;
            }
            __syncwarp();
        }
        float bk = beta;
        if constexpr (ANNEAL) {
            // every lane forms the same sum: each butterfly step adds the same two values in either order
            double e = 0.0;
            for (int k = lane; k < L; k += 32) {
                const int r = k * q + s[k];
                e = __dadd_rn(e, __dsub_rn((double)z[r], (double)h[r]));
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) e = __dadd_rn(e, __shfl_xor_sync(0xffffffffu, e, o));
            const float b0 = betas[t - t0];
            bk = betas[t - t0 + 1];
            w = __dadd_rn(w, __dmul_rn(__dsub_rn((double)bk, (double)b0), __dmul_rn(0.5, e)));
        }
        for (int i = 0; i < L; i++) {
            const float v = lane < q ? (ANNEAL ? annealed_logit(h[i * q + lane], z[i * q + lane], bk)
                                               : beta * z[i * q + lane]) : -INFINITY;
            float m = v;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
            float cum = lane < q ? expf(v - m) : 0.f;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const float y = __shfl_up_sync(0xffffffffu, cum, o);
                if (lane >= o) cum += y;
            }
            const float total = __shfl_sync(0xffffffffu, cum, q - 1);
            // u has 25 significant bits, one more than fp32 holds: u and u * c_{q-1} are exact in double
            const double u = ((double)sample_draw24(key, t, L, i) + 0.5) * 0x1p-24;
            const unsigned hit = __ballot_sync(0xffffffffu, lane < q && u * (double)total < (double)cum);
            const int b = hit ? __ffs(hit) - 1 : q - 1;
            const int a = s[i];
            if (b != a) {
                const float *rb = U + (int64_t)(i * q + b) * Lq;
                const float *ra = U + (int64_t)(i * q + a) * Lq;
#pragma unroll 4
                for (int e = lane; e < Lq; e += 32) z[e] += __ldg(rb + e) - __ldg(ra + e);
                __syncwarp();
                if (lane == 0) s[i] = (uint8_t)b;
                changed++;
            }
            __syncwarp();
        }
        if constexpr (RECORD) {
            const double H = chain_energy(z, h, s, L, q, lane);
            if (H > best) {                     // the same for the whole warp
                best = H;
                best_t = t;
                for (int k = lane; k < L; k += 32) best_codes[c * L + k] = s[k];
            }
        }
    }
    if constexpr (RECORD)
        if (best_t >= 0 && lane == 0) {
            best_energy[c] = best;
            best_sweep[c] = best_t;
        }
    if constexpr (TEMPER)
        if (logw) {                             // the same for the whole warp
            const double H = chain_energy(z, h, s, L, q, lane);
            if (lane == 0) logw[c] = H;
        }
    for (int e = lane; e < Lq; e += 32) zc[e] = z[e];
    for (int k = lane; k < L; k += 32) sc[k] = s[k];
    if (lane == 0 && changed) atomicAdd(changes, changed);
    if constexpr (ANNEAL)
        if (lane == 0) logw[c] = w;
}

// ---- conditional sampling (evc_sampler_create_conditional) -----------------------------------------------------
// Chain c with its context x_c on the clamped sites C samples the free sites F = (F_0 < F_1 < ...) from the Potts model
// with couplings J_FF and fields hc_c,k(a) = h_{F_k}(a) + sum_{j in C} J_{F_k j}(a, x_c,j).  With F = every site the
// fold is h, U_FF is U and the sweep is sample_gibbs_kernel<false>'s, bit for bit.

__device__ __forceinline__ int64_t sample_pair_offset(int i, int j, int L)      // block of the pair i < j in J
{
    return (int64_t)i * L - (int64_t)i * (i + 1) / 2 + (j - i - 1);
}

// hc[c][(k, a)] = h_{F_k}(a), then + J_{F_k j}(a, x_c,j) for every clamped j ascending, each add rounded on its own
__global__ void sample_fold_kernel(const float *__restrict__ h, const float *__restrict__ J,
                                   const int32_t *__restrict__ free_sites, const int32_t *__restrict__ clamped,
                                   const uint8_t *__restrict__ codes, int L, int q, int nf, int64_t n_chains,
                                   float *__restrict__ hc)
{
    const int nfq = nf * q, nc = L - nf;
    const int64_t qq = (int64_t)q * q;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n_chains * nfq;
         e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t c = e / nfq;
        const int r = (int)(e - c * nfq);
        const int k = r / q, a = r - k * q;
        const int i = free_sites[k];
        const uint8_t *x = codes + c * L;
        float acc = h[(int64_t)i * q + a];
        for (int m = 0; m < nc; m++) {
            const int j = clamped[m], b = x[j];
            const int64_t o = i < j ? sample_pair_offset(i, j, L) * qq + a * q + b
                                    : sample_pair_offset(j, i, L) * qq + b * q + a;
            acc = __fadd_rn(acc, J[o]);
        }
        hc[e] = acc;
    }
}

// U_FF: sample_build_u_kernel restricted to the free sites, (nf q) x (nf q), zero diagonal blocks
__global__ void sample_build_uff_kernel(const float *__restrict__ J, const int32_t *__restrict__ free_sites, int L,
                                        int q, int nf, float *__restrict__ U)
{
    const int nfq = nf * q;
    const int r = blockIdx.y;
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nfq) return;
    const int kr = r / q, a = r - kr * q, ke = e / q, b = e - ke * q;
    const int i = free_sites[kr], j = free_sites[ke];
    float v = 0.f;
    if (i < j) v = J[sample_pair_offset(i, j, L) * q * q + a * q + b];
    else if (j < i) v = J[sample_pair_offset(j, i, L) * q * q + b * q + a];
    U[(int64_t)r * nfq + e] = v;
}

// bytes of the CTA's table of free sites and masks, ahead of the chains' rows in shared memory
__host__ __device__ __forceinline__ int64_t conditional_table_bytes(int nf)
{
    return ((int64_t)nf * 8 + 15) / 16 * 16;
}

// sample_gibbs_kernel<false> over the free sites only: Z row (nf q) and free codes in shared memory, refresh from hc_c
// and U_FF rows over free k ascending, counters at the original site index F_k, the draw restricted to allowed[k].
// The free sites and masks are staged once per CTA in shared memory: read from global memory at every site they
// would wait on L2, since the coupling rows a change streams evict them from L1.
// TEMPER: as in sample_gibbs_kernel, the chain's beta is betas[c] and energy[c] (when not null) receives its energy
// over the free sites with hc_c in place of h.  The plain instantiation ignores betas and energy.
// RECORD: as in sample_gibbs_kernel, with that conditional energy; only the free sites of best_codes are written (the
// record's start, evc_sampler_record_best, copies the clamped ones).
template <bool TEMPER, bool RECORD = false>
__global__ void __launch_bounds__(32 * SAMPLE_MAX_WARPS)
sample_conditional_kernel(const float *__restrict__ U, const float *__restrict__ hc, float *__restrict__ Zg,
                          uint8_t *__restrict__ codes, unsigned long long *__restrict__ changes,
                          const int32_t *__restrict__ free_sites, const uint32_t *__restrict__ allowed, int L, int q,
                          int nf, int64_t n_chains, int64_t chain_offset, uint64_t seed, int64_t t0, int sweeps,
                          float beta, int row_bytes, const float *__restrict__ betas, double *__restrict__ energy,
                          double *__restrict__ best_energy, uint8_t *__restrict__ best_codes,
                          int64_t *__restrict__ best_sweep)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    int32_t *site_of = reinterpret_cast<int32_t *>(smem_raw);
    uint32_t *mask_of = reinterpret_cast<uint32_t *>(site_of + nf);
    for (int k = threadIdx.x; k < nf; k += blockDim.x) {
        site_of[k] = free_sites[k];
        mask_of[k] = allowed[k];
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t c = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
    if (c >= n_chains) return;                  // the whole warp: no CTA barrier below
    if constexpr (TEMPER) beta = betas[c];
    const int nfq = nf * q;
    float *z = reinterpret_cast<float *>(smem_raw + conditional_table_bytes(nf) + (size_t)warp * row_bytes);
    uint8_t *s = reinterpret_cast<uint8_t *>(z + nfq);
    float *zc = Zg + c * nfq;
    const float *hcc = hc + c * nfq;
    uint8_t *sc = codes + c * L;
    for (int k = lane; k < nf; k += 32) s[k] = sc[site_of[k]];
    if (t0 % EVC_SAMPLER_REFRESH != 0)
        for (int e = lane; e < nfq; e += 32) z[e] = zc[e];
    __syncwarp();
    const uint64_t key = sample_chain_key(seed, (uint64_t)(chain_offset + c));
    unsigned long long changed = 0;
    double best = 0.0;
    int64_t best_t = -1;
    if constexpr (RECORD) best = best_energy[c];
    for (int64_t t = t0; t < t0 + sweeps; t++) {
        if (t % EVC_SAMPLER_REFRESH == 0) {
            for (int e = lane; e < nfq; e += 32) {
                float acc = hcc[e];
                for (int k = 0; k < nf; k++) acc += U[(int64_t)(k * q + s[k]) * nfq + e];
                z[e] = acc;
            }
            __syncwarp();
        }
        for (int k = 0; k < nf; k++) {
            const uint32_t mask = mask_of[k];
            const bool ok = lane < q && ((mask >> lane) & 1u);
            const float v = ok ? beta * z[k * q + lane] : -INFINITY;
            float m = v;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
            float cum = ok ? expf(v - m) : 0.f;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const float y = __shfl_up_sync(0xffffffffu, cum, o);
                if (lane >= o) cum += y;
            }
            const float total = __shfl_sync(0xffffffffu, cum, q - 1);
            const double u = ((double)sample_draw24(key, t, L, site_of[k]) + 0.5) * 0x1p-24;
            // a disallowed lane repeats the cumulative sum below it, so the smallest hit is always an allowed state
            const unsigned hit = __ballot_sync(0xffffffffu, ok && u * (double)total < (double)cum);
            const int b = hit ? __ffs(hit) - 1 : 31 - __clz(mask);
            const int a = s[k];
            if (b != a) {
                const float *rb = U + (int64_t)(k * q + b) * nfq;
                const float *ra = U + (int64_t)(k * q + a) * nfq;
#pragma unroll 4
                for (int e = lane; e < nfq; e += 32) z[e] += __ldg(rb + e) - __ldg(ra + e);
                __syncwarp();
                if (lane == 0) s[k] = (uint8_t)b;
                changed++;
            }
            __syncwarp();
        }
        if constexpr (RECORD) {
            const double H = chain_energy(z, hcc, s, nf, q, lane);
            if (H > best) {
                best = H;
                best_t = t;
                for (int k = lane; k < nf; k += 32) best_codes[c * L + site_of[k]] = s[k];
            }
        }
    }
    if constexpr (RECORD)
        if (best_t >= 0 && lane == 0) {
            best_energy[c] = best;
            best_sweep[c] = best_t;
        }
    if constexpr (TEMPER)
        if (energy) {                           // the same for the whole warp
            const double H = chain_energy(z, hcc, s, nf, q, lane);
            if (lane == 0) energy[c] = H;
        }
    for (int e = lane; e < nfq; e += 32) zc[e] = z[e];
    for (int k = lane; k < nf; k += 32) sc[site_of[k]] = s[k];
    if (lane == 0 && changed) atomicAdd(changes, changed);
}

// ---- replica exchange (evc_sampler_set_ladder, evc_sampler_temper) ---------------------------------------------------
// Ladder l of the handle is the chains l R .. l R + R - 1, global ladder index ladder_offset + l.  holder[l R + k] is
// the chain (0..R-1 within the ladder) at rung k, rung[] its inverse, chain_beta[c] = ladder[rung[c]] what the tempered
// sweep reads.  heading[c] is the last end of the ladder chain c visited: a chain reaching rung 0 after rung R-1
// completes a round trip.
constexpr int8_t HEAD_NONE = 0, HEAD_UP = 1, HEAD_DOWN = 2;

// the swap stream of ladder g: the key of chain index 2^63 + g, which no chain has (chain indices stay below 2^63)
// and mix, a bijection, gives no other chain's key
__host__ __device__ __forceinline__ uint64_t sample_swap_key(uint64_t seed, uint64_t g)
{
    return sample_chain_key(seed, g | (1ull << 63));
}

// swap round n of every ladder, one thread each: the pairs (k, k + 1), k = n mod 2, n mod 2 + 2, ... in order
__global__ void sample_swap_kernel(const float *__restrict__ ladder, int R, int64_t n_ladders, int64_t ladder_offset,
                                   uint64_t seed, int64_t n, const double *__restrict__ energy,
                                   int32_t *__restrict__ holder, int32_t *__restrict__ rung,
                                   float *__restrict__ chain_beta, int8_t *__restrict__ heading,
                                   long long *__restrict__ trips, unsigned long long *__restrict__ swaps)
{
    const int64_t l = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= n_ladders) return;
    const int64_t base = l * R;
    const uint64_t key = sample_swap_key(seed, (uint64_t)(ladder_offset + l));
    for (int k = (int)(n & 1); k + 1 < R; k += 2) {
        const int x = holder[base + k], y = holder[base + k + 1];
        const double d = __dmul_rn(__dsub_rn((double)ladder[k + 1], (double)ladder[k]),
                                   __dsub_rn(energy[base + x], energy[base + y]));
        const double u = ((double)sample_draw24(key, n, R, k) + 0.5) * 0x1p-24;
        const bool accept = d >= 0.0 || u < exp(d);
        if (swaps) {
            atomicAdd(swaps + k, 1ull);
            if (accept) atomicAdd(swaps + (R - 1) + k, 1ull);
        }
        if (accept) {
            holder[base + k] = y;
            holder[base + k + 1] = x;
            rung[base + x] = k + 1;
            rung[base + y] = k;
            chain_beta[base + x] = ladder[k + 1];
            chain_beta[base + y] = ladder[k];
        }
    }
    const int bottom = holder[base], top = holder[base + R - 1];
    if (heading[base + bottom] == HEAD_DOWN) trips[l]++;
    heading[base + bottom] = HEAD_UP;
    if (heading[base + top] == HEAD_UP) heading[base + top] = HEAD_DOWN;
}

// the start of every ladder: chain l R + k at rung k, only the chain at rung 0 heading up
__global__ void sample_ladder_start_kernel(const float *__restrict__ ladder, int R, int64_t n_chains,
                                           int32_t *__restrict__ holder, int32_t *__restrict__ rung,
                                           float *__restrict__ chain_beta, int8_t *__restrict__ heading,
                                           double *__restrict__ energy, long long *__restrict__ trips)
{
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_chains) return;
    const int k = (int)(c % R);
    holder[c] = k;
    rung[c] = k;
    chain_beta[c] = ladder[k];
    heading[c] = k == 0 ? HEAD_UP : HEAD_NONE;
    energy[c] = 0.0;
    if (k == 0) trips[c / R] = 0;
}

// ---- design (evc_sampler_record_best, evc_sampler_descend) ------------------------------------------------------------

__global__ void sample_record_start_kernel(int64_t n_chains, double *__restrict__ best_energy,
                                           int64_t *__restrict__ best_sweep)
{
    const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_chains) return;
    best_energy[c] = -INFINITY;
    best_sweep[c] = -1;
}

// Zero-temperature descent: the sweep of sample_gibbs_kernel<false> (COND: of sample_conditional_kernel<false>), with
// the same rows in shared memory, refresh rule and change update, whose draw is replaced by the single-site argmax in
// fp32.  Per site, m = the max of Z_k(a) over the allowed a (COND: the mask; plain: every a < q); s_k stays if it is
// allowed and Z_k(s_k) == m, else becomes the smallest allowed a with Z_k(a) == m.  No uniforms: the step is a function
// of Z and s only.  settled[c] (when not null) = 1 if the call's last sweep changed no site of chain c, else 0.
template <bool COND>
__global__ void __launch_bounds__(32 * SAMPLE_MAX_WARPS)
sample_descent_kernel(const float *__restrict__ U, const float *__restrict__ h, float *__restrict__ Zg,
                      uint8_t *__restrict__ codes, unsigned long long *__restrict__ changes,
                      const int32_t *__restrict__ free_sites, const uint32_t *__restrict__ allowed, int L, int q,
                      int nf, int64_t n_chains, int64_t t0, int sweeps, int row_bytes, bool refresh_first,
                      uint8_t *__restrict__ settled)
{
    extern __shared__ __align__(16) unsigned char smem_raw[];
    int32_t *site_of = reinterpret_cast<int32_t *>(smem_raw);
    uint32_t *mask_of = reinterpret_cast<uint32_t *>(site_of + nf);
    if constexpr (COND) {
        for (int k = threadIdx.x; k < nf; k += blockDim.x) {
            site_of[k] = free_sites[k];
            mask_of[k] = allowed[k];
        }
        __syncthreads();
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t c = (int64_t)blockIdx.x * (blockDim.x >> 5) + warp;
    if (c >= n_chains) return;                  // the whole warp: no CTA barrier below
    const int n = COND ? nf : L, nq = n * q;
    float *z = reinterpret_cast<float *>(smem_raw + (COND ? conditional_table_bytes(nf) : 0) +
                                         (size_t)warp * row_bytes);
    uint8_t *s = reinterpret_cast<uint8_t *>(z + nq);
    float *zc = Zg + c * nq;
    const float *hr = COND ? h + c * nq : h;    // COND: the chain's folded fields hc_c
    uint8_t *sc = codes + c * L;
    for (int k = lane; k < n; k += 32) s[k] = sc[COND ? site_of[k] : k];
    if (t0 % EVC_SAMPLER_REFRESH != 0 && !refresh_first)
        for (int e = lane; e < nq; e += 32) z[e] = zc[e];
    __syncwarp();
    unsigned long long changed = 0, before = 0;
    for (int64_t t = t0; t < t0 + sweeps; t++) {
        if (t % EVC_SAMPLER_REFRESH == 0 || (refresh_first && t == t0)) {
            for (int e = lane; e < nq; e += 32) {
                float acc = hr[e];
                for (int j = 0; j < n; j++) acc += U[(int64_t)(j * q + s[j]) * nq + e];
                z[e] = acc;
            }
            __syncwarp();
        }
        before = changed;
        for (int k = 0; k < n; k++) {
            const bool ok = lane < q && (!COND || ((mask_of[k] >> lane) & 1u));
            const float v = ok ? z[k * q + lane] : -INFINITY;
            float m = v;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
            const unsigned top = __ballot_sync(0xffffffffu, ok && v == m);
            const int a = s[k];
            const int b = ((top >> a) & 1u) || !top ? a : __ffs(top) - 1;
            if (b != a) {
                const float *rb = U + (int64_t)(k * q + b) * nq;
                const float *ra = U + (int64_t)(k * q + a) * nq;
#pragma unroll 4
                for (int e = lane; e < nq; e += 32) z[e] += __ldg(rb + e) - __ldg(ra + e);
                __syncwarp();
                if (lane == 0) s[k] = (uint8_t)b;
                changed++;
            }
            __syncwarp();
        }
    }
    for (int e = lane; e < nq; e += 32) zc[e] = z[e];
    for (int k = lane; k < n; k += 32) sc[COND ? site_of[k] : k] = s[k];
    if (lane == 0 && changed) atomicAdd(changes, changed);
    if (lane == 0 && settled) settled[c] = changed == before ? 1 : 0;
}

}  // namespace evc

using namespace evc;

struct evc_sampler {
    int device = 0;
    int L = 0, q = 0;
    int64_t n_chains = 0, chain_offset = 0;
    uint64_t seed = 0;
    int64_t t = 0;                      // global sweep index of the next sweep
    bool refresh_next = false;          // evc_sampler_set_model: recompute Z before the next sweep
    float *U = nullptr, *h = nullptr, *Z = nullptr;
    uint8_t *codes = nullptr;
    unsigned long long *changes = nullptr;
    float *betas = nullptr;             // evc_sampler_anneal: device copy of the last schedule
    int64_t betas_cap = 0;
    // evc_sampler_create_conditional: U is U_FF, h is unused, Z holds nf q floats per chain
    bool conditional = false;
    int nf = 0;
    int32_t *free_sites = nullptr;      // nf ascending site indices
    uint32_t *allowed = nullptr;        // nf allowed-state masks
    float *hc = nullptr;                // n_chains x nf q folded fields
    // evc_sampler_set_ladder: R > 0 once a ladder is set
    int R = 0;
    int64_t swap_interval = 0;
    std::vector<float> ladder_host;
    float *ladder = nullptr;            // R betas
    float *chain_beta = nullptr;        // n_chains: the beta of the rung each chain holds
    int32_t *holder = nullptr, *rung = nullptr;
    int8_t *heading = nullptr;
    double *energy = nullptr;           // n_chains: the energies of the last swap round
    long long *trips = nullptr;         // n_chains / R round trips
    // evc_sampler_record_best: non-null once a record is started; run and temper then record
    double *best_energy = nullptr;      // n_chains
    uint8_t *best_codes = nullptr;      // n_chains x L
    int64_t *best_sweep = nullptr;      // n_chains
};

static void sampler_free(evc_sampler *s)
{
    cudaFree(s->ladder);
    cudaFree(s->chain_beta);
    cudaFree(s->holder);
    cudaFree(s->rung);
    cudaFree(s->heading);
    cudaFree(s->energy);
    cudaFree(s->trips);
    cudaFree(s->U);
    cudaFree(s->h);
    cudaFree(s->Z);
    cudaFree(s->codes);
    cudaFree(s->changes);
    cudaFree(s->betas);
    cudaFree(s->free_sites);
    cudaFree(s->allowed);
    cudaFree(s->hc);
    cudaFree(s->best_energy);
    cudaFree(s->best_codes);
    cudaFree(s->best_sweep);
    delete s;
}

// the number of site changes counted on the device since the last reset, when asked for (synchronises `st`)
static int read_changes(evc_sampler *s, int64_t *changes_out, cudaStream_t st)
{
    if (changes_out) {
        unsigned long long n = 0;
        EVC_CUDA(cudaMemcpyAsync(&n, s->changes, sizeof(n), cudaMemcpyDeviceToHost, st));
        EVC_CUDA(cudaStreamSynchronize(st));
        *changes_out = (int64_t)n;
    }
    return 0;
}

// one launch of sweeps >= 1 sweeps of every chain from the handle's sweep index on: plain (beta), annealed (betas,
// logw) or tempered (betas = the chains' betas, logw = the energies to write or null); RECORD when a record is kept
template <bool ANNEAL, bool TEMPER, bool RECORD>
static int gibbs_launch_as(evc_sampler *s, int32_t sweeps, float beta, const float *betas, double *logw,
                           cudaStream_t st)
{
    const int row_bytes = (int)sample_row_bytes(s->L, s->q);
    const int warps = std::min<int64_t>(std::min(SAMPLE_MAX_WARPS, SAMPLE_SMEM_MAX / row_bytes), s->n_chains);
    const size_t smem = (size_t)warps * row_bytes;
    EVC_CUDA(cudaFuncSetAttribute(sample_gibbs_kernel<ANNEAL, TEMPER, RECORD>,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    sample_gibbs_kernel<ANNEAL, TEMPER, RECORD><<<(unsigned)ceil_div(s->n_chains, warps), 32 * warps, smem, st>>>(
        s->U, s->h, s->Z, s->codes, s->changes, s->L, s->q, s->n_chains, s->chain_offset, s->seed, s->t, sweeps,
        beta, row_bytes, s->refresh_next, betas, logw, s->best_energy, s->best_codes, s->best_sweep);
    EVC_KERNEL_CHECK();
    s->t += sweeps;
    s->refresh_next = false;
    return 0;
}

template <bool ANNEAL, bool TEMPER>
static int gibbs_launch(evc_sampler *s, int32_t sweeps, float beta, const float *betas, double *logw, cudaStream_t st)
{
    if constexpr (!ANNEAL)
        if (s->best_energy) return gibbs_launch_as<false, TEMPER, true>(s, sweeps, beta, betas, logw, st);
    return gibbs_launch_as<ANNEAL, TEMPER, false>(s, sweeps, beta, betas, logw, st);
}

// one launch of sweeps >= 1 sweeps of the free sites of every chain of a conditional handle, plain (beta) or
// tempered (betas, energy as in gibbs_launch)
template <bool TEMPER, bool RECORD>
static int conditional_launch_as(evc_sampler *s, int32_t sweeps, float beta, const float *betas, double *energy,
                                 cudaStream_t st)
{
    const int row_bytes = (int)sample_row_bytes(s->nf, s->q);
    const int64_t table = conditional_table_bytes(s->nf);
    const int warps = std::min<int64_t>(std::min<int64_t>(SAMPLE_MAX_WARPS, (SAMPLE_SMEM_MAX - table) / row_bytes),
                                        s->n_chains);
    const size_t smem = (size_t)table + (size_t)warps * row_bytes;
    EVC_CUDA(cudaFuncSetAttribute(sample_conditional_kernel<TEMPER, RECORD>,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    sample_conditional_kernel<TEMPER, RECORD><<<(unsigned)ceil_div(s->n_chains, warps), 32 * warps, smem, st>>>(
        s->U, s->hc, s->Z, s->codes, s->changes, s->free_sites, s->allowed, s->L, s->q, s->nf, s->n_chains,
        s->chain_offset, s->seed, s->t, sweeps, beta, row_bytes, betas, energy, s->best_energy, s->best_codes,
        s->best_sweep);
    EVC_KERNEL_CHECK();
    s->t += sweeps;
    return 0;
}

template <bool TEMPER>
static int conditional_launch(evc_sampler *s, int32_t sweeps, float beta, const float *betas, double *energy,
                              cudaStream_t st)
{
    if (s->best_energy) return conditional_launch_as<TEMPER, true>(s, sweeps, beta, betas, energy, st);
    return conditional_launch_as<TEMPER, false>(s, sweeps, beta, betas, energy, st);
}

// one launch of sweeps >= 1 descent sweeps of every chain (of the free sites of a conditional handle)
template <bool COND>
static int descent_launch(evc_sampler *s, int32_t sweeps, uint8_t *settled, cudaStream_t st)
{
    const int n = COND ? s->nf : s->L;
    const int row_bytes = (int)sample_row_bytes(n, s->q);
    const int64_t table = COND ? conditional_table_bytes(s->nf) : 0;
    const int warps = std::min<int64_t>(std::min<int64_t>(SAMPLE_MAX_WARPS, (SAMPLE_SMEM_MAX - table) / row_bytes),
                                        s->n_chains);
    const size_t smem = (size_t)table + (size_t)warps * row_bytes;
    EVC_CUDA(cudaFuncSetAttribute(sample_descent_kernel<COND>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)smem));
    sample_descent_kernel<COND><<<(unsigned)ceil_div(s->n_chains, warps), 32 * warps, smem, st>>>(
        s->U, COND ? s->hc : s->h, s->Z, s->codes, s->changes, s->free_sites, s->allowed, s->L, s->q, s->nf,
        s->n_chains, s->t, sweeps, row_bytes, s->refresh_next, settled);
    EVC_KERNEL_CHECK();
    s->t += sweeps;
    s->refresh_next = false;
    return 0;
}

// `sweeps` sweeps of every chain from the handle's sweep index on, plain (beta) or annealed (betas, logw)
template <bool ANNEAL>
static int sampler_sweeps(evc_sampler *s, int32_t sweeps, float beta, const float *betas, double *logw,
                          int64_t *changes_out, cudaStream_t st)
{
    EVC_CUDA(cudaMemsetAsync(s->changes, 0, sizeof(unsigned long long), st));
    if (sweeps > 0 && gibbs_launch<ANNEAL, false>(s, sweeps, beta, betas, logw, st)) return 1;
    return read_changes(s, changes_out, st);
}

// `sweeps` sweeps of the free sites of every chain of a conditional handle
static int conditional_sweeps(evc_sampler *s, int32_t sweeps, float beta, int64_t *changes_out, cudaStream_t st)
{
    EVC_CUDA(cudaMemsetAsync(s->changes, 0, sizeof(unsigned long long), st));
    if (sweeps > 0 && conditional_launch<false>(s, sweeps, beta, nullptr, nullptr, st)) return 1;
    return read_changes(s, changes_out, st);
}

extern "C" {

int evc_sampler_create(evc_sampler_t **out, const float *d_x, int32_t L, int32_t q, const uint8_t *init,
                       int64_t n_chains, int64_t chain_offset, uint64_t seed, int32_t device)
{
    const std::string name = "evc_sampler_create";
    if (!out || !d_x) { set_error(name + ": null pointer"); return 1; }
    *out = nullptr;
    if (q < 2 || q > 32) {
        set_error(name + ": unsupported number of states q=" + std::to_string(q) + " (2 <= q <= 32)");
        return 1;
    }
    if (L < 2) { set_error(name + ": need L >= 2 sites"); return 1; }
    if (sample_row_bytes(L, q) > SAMPLE_SMEM_MAX) {
        set_error(name + ": L=" + std::to_string(L) + ", q=" + std::to_string(q) + " is too large: one chain's " +
                  "field row (4 L q bytes) and its L codes must fit the " + std::to_string(SAMPLE_SMEM_MAX) +
                  " bytes of shared memory of one CTA, i.e. L q up to about 58 000");
        return 1;
    }
    if (n_chains < 1 || n_chains > (INT64_MAX / 4) / ((int64_t)L * q)) {
        set_error(name + ": n_chains must be >= 1 (got " + std::to_string(n_chains) + ") and n_chains L q < 2^61");
        return 1;
    }
    if (chain_offset < 0 || chain_offset > INT64_MAX - n_chains) {
        set_error(name + ": chain_offset must be >= 0 and chain_offset + n_chains < 2^63");
        return 1;
    }
    if (init) {
        for (int64_t e = 0; e < n_chains * L; e++) {
            if (init[e] >= q) {
                set_error(name + ": init code " + std::to_string(init[e]) + " at chain " + std::to_string(e / L) +
                          ", site " + std::to_string(e % L) + " out of range (valid: 0.." + std::to_string(q - 1) + ")");
                return 1;
            }
        }
    }
    EVC_CUDA(cudaSetDevice(device));
    evc_sampler *s = new (std::nothrow) evc_sampler;
    if (!s) { set_error(name + ": out of host memory"); return 1; }
    s->device = device;
    s->L = L;
    s->q = q;
    s->n_chains = n_chains;
    s->chain_offset = chain_offset;
    s->seed = seed;
    const int64_t Lq = (int64_t)L * q;
    if (cudaMalloc(&s->U, (size_t)Lq * Lq * sizeof(float)) != cudaSuccess ||
        cudaMalloc(&s->h, (size_t)Lq * sizeof(float)) != cudaSuccess ||
        cudaMalloc(&s->Z, (size_t)n_chains * Lq * sizeof(float)) != cudaSuccess ||
        cudaMalloc(&s->codes, (size_t)n_chains * L) != cudaSuccess ||
        cudaMalloc(&s->changes, sizeof(unsigned long long)) != cudaSuccess) {
        set_error(name + ": device allocation failed: " + cudaGetErrorString(cudaGetLastError()));
        sampler_free(s);
        return 1;
    }
    bool ok = cudaMemcpy(s->h, d_x, (size_t)Lq * sizeof(float), cudaMemcpyDeviceToDevice) == cudaSuccess;
    if (ok) {
        sample_build_u_kernel<<<dim3((unsigned)ceil_div(Lq, 256), (unsigned)Lq), 256>>>(d_x + Lq, L, q, s->U);
        ok = cudaGetLastError() == cudaSuccess;
    }
    if (ok && init) {
        ok = cudaMemcpy(s->codes, init, (size_t)n_chains * L, cudaMemcpyHostToDevice) == cudaSuccess;
    } else if (ok) {
        sample_uniform_start_kernel<<<(unsigned)ceil_div(n_chains * L, 256), 256>>>(s->codes, n_chains, chain_offset,
                                                                                    seed, L, q);
        ok = cudaGetLastError() == cudaSuccess;
    }
    if (ok) ok = cudaDeviceSynchronize() == cudaSuccess;
    if (!ok) {
        set_error(name + ": building the couplings or the start failed: " + cudaGetErrorString(cudaGetLastError()));
        sampler_free(s);
        return 1;
    }
    *out = s;
    return 0;
}

int evc_sampler_create_conditional(evc_sampler_t **out, const float *d_x, int32_t L, int32_t q,
                                   const int32_t *free_sites, int32_t nf, const uint32_t *allowed,
                                   const uint8_t *init, int64_t n_chains, int64_t chain_offset, uint64_t seed,
                                   int32_t device)
{
    const std::string name = "evc_sampler_create_conditional";
    if (!out || !d_x || !free_sites) { set_error(name + ": null pointer"); return 1; }
    *out = nullptr;
    if (q < 2 || q > 32) {
        set_error(name + ": unsupported number of states q=" + std::to_string(q) + " (2 <= q <= 32)");
        return 1;
    }
    if (L < 2) { set_error(name + ": need L >= 2 sites"); return 1; }
    if (nf < 1 || nf > L) {
        set_error(name + ": need 1 <= nf <= L free sites (got nf=" + std::to_string(nf) + ", L=" + std::to_string(L) +
                  ")");
        return 1;
    }
    for (int32_t k = 0; k < nf; k++) {
        if (free_sites[k] < 0 || free_sites[k] >= L || (k > 0 && free_sites[k] <= free_sites[k - 1])) {
            set_error(name + ": free_sites must be strictly ascending site indices in [0, L): free_sites[" +
                      std::to_string(k) + "] = " + std::to_string(free_sites[k]));
            return 1;
        }
    }
    const uint32_t full = q == 32 ? 0xffffffffu : (1u << q) - 1u;
    if (allowed) {
        for (int32_t k = 0; k < nf; k++) {
            if (allowed[k] == 0 || (allowed[k] & ~full)) {
                set_error(name + ": allowed[" + std::to_string(k) + "] = " + std::to_string(allowed[k]) +
                          " must be a non-zero mask of states below q=" + std::to_string(q));
                return 1;
            }
        }
    }
    if (!init && nf < L) {
        set_error(name + ": init is required when sites are clamped (nf < L): it holds each chain's context");
        return 1;
    }
    if (conditional_table_bytes(nf) + sample_row_bytes(nf, q) > SAMPLE_SMEM_MAX) {
        set_error(name + ": nf=" + std::to_string(nf) + ", q=" + std::to_string(q) + " is too large: one chain's " +
                  "field row over the free sites (4 nf q bytes), its nf codes and the CTA's table of free sites and " +
                  "masks (8 nf bytes) must fit the " + std::to_string(SAMPLE_SMEM_MAX) +
                  " bytes of shared memory of one CTA, i.e. nf q up to about 58 000");
        return 1;
    }
    if (n_chains < 1 || n_chains > (INT64_MAX / 8) / ((int64_t)L * q)) {
        set_error(name + ": n_chains must be >= 1 (got " + std::to_string(n_chains) + ") and n_chains L q < 2^60");
        return 1;
    }
    if (chain_offset < 0 || chain_offset > INT64_MAX - n_chains) {
        set_error(name + ": chain_offset must be >= 0 and chain_offset + n_chains < 2^63");
        return 1;
    }
    if (init) {
        for (int64_t e = 0; e < n_chains * L; e++) {
            if (init[e] >= q) {
                set_error(name + ": init code " + std::to_string(init[e]) + " at chain " + std::to_string(e / L) +
                          ", site " + std::to_string(e % L) + " out of range (valid: 0.." + std::to_string(q - 1) + ")");
                return 1;
            }
        }
    }
    std::vector<int32_t> clamped;
    for (int32_t i = 0, k = 0; i < L; i++) {
        if (k < nf && free_sites[k] == i) k++;
        else clamped.push_back(i);
    }
    std::vector<uint32_t> masks(nf, full);
    if (allowed) std::copy(allowed, allowed + nf, masks.begin());
    EVC_CUDA(cudaSetDevice(device));
    evc_sampler *s = new (std::nothrow) evc_sampler;
    if (!s) { set_error(name + ": out of host memory"); return 1; }
    s->device = device;
    s->L = L;
    s->q = q;
    s->n_chains = n_chains;
    s->chain_offset = chain_offset;
    s->seed = seed;
    s->conditional = true;
    s->nf = nf;
    const int64_t nfq = (int64_t)nf * q;
    int32_t *d_clamped = nullptr;
    if (cudaMalloc(&s->U, (size_t)nfq * nfq * sizeof(float)) != cudaSuccess ||
        cudaMalloc(&s->hc, (size_t)n_chains * nfq * sizeof(float)) != cudaSuccess ||
        cudaMalloc(&s->Z, (size_t)n_chains * nfq * sizeof(float)) != cudaSuccess ||
        cudaMalloc(&s->codes, (size_t)n_chains * L) != cudaSuccess ||
        cudaMalloc(&s->changes, sizeof(unsigned long long)) != cudaSuccess ||
        cudaMalloc(&s->free_sites, (size_t)nf * sizeof(int32_t)) != cudaSuccess ||
        cudaMalloc(&s->allowed, (size_t)nf * sizeof(uint32_t)) != cudaSuccess ||
        cudaMalloc(&d_clamped, std::max<size_t>(clamped.size(), 1) * sizeof(int32_t)) != cudaSuccess) {
        set_error(name + ": device allocation failed: " + cudaGetErrorString(cudaGetLastError()));
        cudaFree(d_clamped);
        sampler_free(s);
        return 1;
    }
    bool ok = cudaMemcpy(s->free_sites, free_sites, (size_t)nf * sizeof(int32_t), cudaMemcpyHostToDevice) ==
                  cudaSuccess &&
              cudaMemcpy(s->allowed, masks.data(), (size_t)nf * sizeof(uint32_t), cudaMemcpyHostToDevice) ==
                  cudaSuccess &&
              (clamped.empty() || cudaMemcpy(d_clamped, clamped.data(), clamped.size() * sizeof(int32_t),
                                             cudaMemcpyHostToDevice) == cudaSuccess);
    if (ok && init) {
        ok = cudaMemcpy(s->codes, init, (size_t)n_chains * L, cudaMemcpyHostToDevice) == cudaSuccess;
    } else if (ok) {
        sample_uniform_start_kernel<<<(unsigned)ceil_div(n_chains * L, 256), 256>>>(s->codes, n_chains, chain_offset,
                                                                                    seed, L, q);
        ok = cudaGetLastError() == cudaSuccess;
    }
    if (ok) {
        sample_build_uff_kernel<<<dim3((unsigned)ceil_div(nfq, 256), (unsigned)nfq), 256>>>(d_x + (int64_t)L * q,
                                                                                            s->free_sites, L, q, nf,
                                                                                            s->U);
        const int64_t blocks = std::min<int64_t>(ceil_div(n_chains * nfq, 256), 1 << 20);
        sample_fold_kernel<<<(unsigned)blocks, 256>>>(d_x, d_x + (int64_t)L * q, s->free_sites, d_clamped, s->codes,
                                                      L, q, nf, n_chains, s->hc);
        ok = cudaGetLastError() == cudaSuccess;
    }
    if (ok) ok = cudaDeviceSynchronize() == cudaSuccess;
    cudaFree(d_clamped);
    if (!ok) {
        set_error(name + ": building the couplings, the start or the fields failed: " +
                  cudaGetErrorString(cudaGetLastError()));
        sampler_free(s);
        return 1;
    }
    *out = s;
    return 0;
}

int evc_sampler_conditional_fields(const evc_sampler_t *s, float *d_out, void *stream)
{
    if (!s || !d_out) { set_error("evc_sampler_conditional_fields: null pointer"); return 1; }
    if (!s->conditional) {
        set_error("evc_sampler_conditional_fields: the handle is not conditional (evc_sampler_create_conditional)");
        return 1;
    }
    EVC_CUDA(cudaSetDevice(s->device));
    EVC_CUDA(cudaMemcpyAsync(d_out, s->hc, (size_t)s->n_chains * s->nf * s->q * sizeof(float),
                             cudaMemcpyDeviceToDevice, reinterpret_cast<cudaStream_t>(stream)));
    return 0;
}

int evc_sampler_run(evc_sampler_t *s, int32_t sweeps, float beta, int64_t *changes_out, void *stream)
{
    if (!s) { set_error("evc_sampler_run: null handle"); return 1; }
    if (sweeps < 0) { set_error("evc_sampler_run: sweeps must be >= 0"); return 1; }
    if (!isfinite(beta)) { set_error("evc_sampler_run: beta must be finite"); return 1; }
    EVC_CUDA(cudaSetDevice(s->device));
    if (s->conditional)
        return conditional_sweeps(s, sweeps, beta, changes_out, reinterpret_cast<cudaStream_t>(stream));
    return sampler_sweeps<false>(s, sweeps, beta, nullptr, nullptr, changes_out,
                                 reinterpret_cast<cudaStream_t>(stream));
}

int evc_sampler_anneal(evc_sampler_t *s, const float *betas, int32_t K, double *d_logw, int64_t *changes_out,
                       void *stream)
{
    const std::string name = "evc_sampler_anneal";
    if (K < 0) { set_error(name + ": K must be >= 0 (got " + std::to_string(K) + ")"); return 1; }
    if (!betas || !d_logw) { set_error(name + ": null pointer"); return 1; }
    for (int32_t k = 0; k <= K; k++) {
        if (!isfinite(betas[k])) {
            set_error(name + ": betas[" + std::to_string(k) + "] is not finite");
            return 1;
        }
    }
    if (!s) { set_error(name + ": null handle"); return 1; }
    if (s->conditional) {
        set_error(name + ": not supported on a conditional sampler (evc_sampler_create_conditional)");
        return 1;
    }
    if (s->R) {
        set_error(name + ": not supported on a tempered sampler (evc_sampler_set_ladder)");
        return 1;
    }
    if (s->best_energy) {
        set_error(name + ": not supported on a handle that records its best states (evc_sampler_record_best)");
        return 1;
    }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    EVC_CUDA(cudaSetDevice(s->device));
    if (K > 0) {
        if (s->betas_cap < (int64_t)K + 1) {
            // cudaFree waits for the kernels that may still read the old schedule
            EVC_CUDA(cudaFree(s->betas));
            s->betas = nullptr;
            s->betas_cap = 0;
            EVC_CUDA(cudaMalloc(&s->betas, ((size_t)K + 1) * sizeof(float)));
            s->betas_cap = (int64_t)K + 1;
        }
        // stream-ordered after the previous call's kernel, which read the last schedule
        EVC_CUDA(cudaMemcpyAsync(s->betas, betas, ((size_t)K + 1) * sizeof(float), cudaMemcpyHostToDevice, st));
    }
    return sampler_sweeps<true>(s, K, 0.f, s->betas, d_logw, changes_out, st);
}

int evc_sampler_set_model(evc_sampler_t *s, const float *d_x, void *stream)
{
    if (!s || !d_x) { set_error("evc_sampler_set_model: null pointer"); return 1; }
    if (s->conditional) {
        set_error("evc_sampler_set_model: not supported on a conditional sampler (evc_sampler_create_conditional)");
        return 1;
    }
    if (s->R) {
        set_error("evc_sampler_set_model: not supported on a tempered sampler (evc_sampler_set_ladder)");
        return 1;
    }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int64_t Lq = (int64_t)s->L * s->q;
    EVC_CUDA(cudaSetDevice(s->device));
    EVC_CUDA(cudaMemcpyAsync(s->h, d_x, (size_t)Lq * sizeof(float), cudaMemcpyDeviceToDevice, st));
    sample_build_u_kernel<<<dim3((unsigned)ceil_div(Lq, 256), (unsigned)Lq), 256, 0, st>>>(d_x + Lq, s->L, s->q, s->U);
    EVC_KERNEL_CHECK();
    s->refresh_next = true;
    return 0;
}

int evc_sampler_set_ladder(evc_sampler_t *s, const float *betas, int32_t R, int64_t swap_interval)
{
    const std::string name = "evc_sampler_set_ladder";
    if (!s || !betas) { set_error(name + ": null pointer"); return 1; }
    if (R < 2) { set_error(name + ": a ladder needs R >= 2 rungs (got " + std::to_string(R) + ")"); return 1; }
    for (int32_t k = 0; k < R; k++) {
        if (!isfinite(betas[k]) || (k == 0 && !(betas[0] >= 0.f)) || (k > 0 && !(betas[k] > betas[k - 1]))) {
            set_error(name + ": betas must be finite and strictly ascending from betas[0] >= 0: betas[" +
                      std::to_string(k) + "] = " + std::to_string(betas[k]));
            return 1;
        }
    }
    if (swap_interval < 1) {
        set_error(name + ": swap_interval must be >= 1 (got " + std::to_string(swap_interval) + ")");
        return 1;
    }
    if (s->n_chains % R != 0) {
        set_error(name + ": n_chains = " + std::to_string(s->n_chains) + " is not a multiple of R = " +
                  std::to_string(R) + ": the handle holds whole ladders");
        return 1;
    }
    if (s->chain_offset % R != 0) {
        set_error(name + ": chain_offset = " + std::to_string(s->chain_offset) + " is not a multiple of R = " +
                  std::to_string(R) + ": ladders start at multiples of R");
        return 1;
    }
    if (s->R) {
        if (s->R == R && s->swap_interval == swap_interval && std::equal(betas, betas + R, s->ladder_host.begin()))
            return 0;
        set_error(name + ": the handle already has a different ladder; a ladder is set once per handle");
        return 1;
    }
    EVC_CUDA(cudaSetDevice(s->device));
    if (s->conditional && s->nf < s->L) {
        // swaps exchange states between chains, so the chains of one ladder must sample one conditional model
        std::vector<uint8_t> x((size_t)s->n_chains * s->L);
        EVC_CUDA(cudaMemcpy(x.data(), s->codes, x.size(), cudaMemcpyDeviceToHost));
        std::vector<bool> is_free(s->L, false);
        std::vector<int32_t> sites(s->nf);
        EVC_CUDA(cudaMemcpy(sites.data(), s->free_sites, (size_t)s->nf * sizeof(int32_t), cudaMemcpyDeviceToHost));
        for (int32_t k : sites) is_free[k] = true;
        for (int64_t c = 0; c < s->n_chains; c++) {
            const uint8_t *a = x.data() + (size_t)c * s->L, *b = x.data() + (size_t)(c - c % R) * s->L;
            for (int j = 0; j < s->L; j++) {
                if (!is_free[j] && a[j] != b[j]) {
                    set_error(name + ": chain " + std::to_string(c) + " and chain " + std::to_string(c - c % R) +
                              " of one ladder have different contexts (clamped site " + std::to_string(j) +
                              "): every chain of a ladder must share its clamped sites");
                    return 1;
                }
            }
        }
    }
    const int64_t n = s->n_chains;
    if (cudaMalloc(&s->ladder, (size_t)R * sizeof(float)) != cudaSuccess ||
        cudaMalloc(&s->chain_beta, (size_t)n * sizeof(float)) != cudaSuccess ||
        cudaMalloc(&s->holder, (size_t)n * sizeof(int32_t)) != cudaSuccess ||
        cudaMalloc(&s->rung, (size_t)n * sizeof(int32_t)) != cudaSuccess ||
        cudaMalloc(&s->heading, (size_t)n) != cudaSuccess ||
        cudaMalloc(&s->energy, (size_t)n * sizeof(double)) != cudaSuccess ||
        cudaMalloc(&s->trips, (size_t)(n / R) * sizeof(long long)) != cudaSuccess) {
        set_error(name + ": device allocation failed: " + cudaGetErrorString(cudaGetLastError()));
        for (void **p : {(void **)&s->ladder, (void **)&s->chain_beta, (void **)&s->holder, (void **)&s->rung,
                         (void **)&s->heading, (void **)&s->energy, (void **)&s->trips}) {
            cudaFree(*p);
            *p = nullptr;
        }
        return 1;
    }
    EVC_CUDA(cudaMemcpy(s->ladder, betas, (size_t)R * sizeof(float), cudaMemcpyHostToDevice));
    sample_ladder_start_kernel<<<(unsigned)ceil_div(n, 256), 256>>>(s->ladder, R, n, s->holder, s->rung,
                                                                   s->chain_beta, s->heading, s->energy, s->trips);
    EVC_KERNEL_CHECK();
    EVC_CUDA(cudaDeviceSynchronize());
    s->R = R;
    s->swap_interval = swap_interval;
    s->ladder_host.assign(betas, betas + R);
    return 0;
}

int evc_sampler_temper(evc_sampler_t *s, int32_t sweeps, int64_t *d_swaps, int64_t *changes_out, void *stream)
{
    const std::string name = "evc_sampler_temper";
    if (!s) { set_error(name + ": null handle"); return 1; }
    if (sweeps < 0) { set_error(name + ": sweeps must be >= 0"); return 1; }
    if (!s->R) { set_error(name + ": the handle has no ladder (evc_sampler_set_ladder)"); return 1; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    EVC_CUDA(cudaSetDevice(s->device));
    EVC_CUDA(cudaMemsetAsync(s->changes, 0, sizeof(unsigned long long), st));
    const int64_t n_ladders = s->n_chains / s->R;
    for (int32_t done = 0; done < sweeps;) {
        // up to and including the next sweep t with (t + 1) % swap_interval == 0
        const int64_t to_round = s->swap_interval - s->t % s->swap_interval;
        const int32_t k = (int32_t)std::min<int64_t>(sweeps - done, to_round);
        double *energy = k == to_round ? s->energy : nullptr;
        const int rc = s->conditional ? conditional_launch<true>(s, k, 0.f, s->chain_beta, energy, st)
                                      : gibbs_launch<false, true>(s, k, 0.f, s->chain_beta, energy, st);
        if (rc) return 1;
        done += k;
        if (energy) {
            sample_swap_kernel<<<(unsigned)ceil_div(n_ladders, 128), 128, 0, st>>>(
                s->ladder, s->R, n_ladders, s->chain_offset / s->R, s->seed, s->t / s->swap_interval - 1, s->energy,
                s->holder, s->rung, s->chain_beta, s->heading, s->trips,
                reinterpret_cast<unsigned long long *>(d_swaps));
            EVC_KERNEL_CHECK();
        }
    }
    return read_changes(s, changes_out, st);
}

int evc_sampler_ladder_state(const evc_sampler_t *s, int32_t *d_rung, double *d_energy, int64_t *d_round_trips,
                             void *stream)
{
    const std::string name = "evc_sampler_ladder_state";
    if (!s) { set_error(name + ": null handle"); return 1; }
    if (!s->R) { set_error(name + ": the handle has no ladder (evc_sampler_set_ladder)"); return 1; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const size_t n = (size_t)s->n_chains;
    EVC_CUDA(cudaSetDevice(s->device));
    if (d_rung) EVC_CUDA(cudaMemcpyAsync(d_rung, s->rung, n * sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
    if (d_energy) EVC_CUDA(cudaMemcpyAsync(d_energy, s->energy, n * sizeof(double), cudaMemcpyDeviceToDevice, st));
    if (d_round_trips)
        EVC_CUDA(cudaMemcpyAsync(d_round_trips, s->trips, n / s->R * sizeof(int64_t), cudaMemcpyDeviceToDevice, st));
    return 0;
}

int evc_sampler_record_best(evc_sampler_t *s, void *stream)
{
    const std::string name = "evc_sampler_record_best";
    if (!s) { set_error(name + ": null handle"); return 1; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const size_t n = (size_t)s->n_chains;
    EVC_CUDA(cudaSetDevice(s->device));
    if (!s->best_energy) {
        if (cudaMalloc(&s->best_energy, n * sizeof(double)) != cudaSuccess ||
            cudaMalloc(&s->best_codes, n * s->L) != cudaSuccess ||
            cudaMalloc(&s->best_sweep, n * sizeof(int64_t)) != cudaSuccess) {
            set_error(name + ": device allocation failed: " + cudaGetErrorString(cudaGetLastError()));
            for (void **p : {(void **)&s->best_energy, (void **)&s->best_codes, (void **)&s->best_sweep}) {
                cudaFree(*p);
                *p = nullptr;
            }
            return 1;
        }
    }
    // the current codes: a conditional sweep writes only the free sites of a new record
    EVC_CUDA(cudaMemcpyAsync(s->best_codes, s->codes, n * s->L, cudaMemcpyDeviceToDevice, st));
    sample_record_start_kernel<<<(unsigned)ceil_div(s->n_chains, 256), 256, 0, st>>>(s->n_chains, s->best_energy,
                                                                                     s->best_sweep);
    EVC_KERNEL_CHECK();
    return 0;
}

int evc_sampler_best(const evc_sampler_t *s, double *d_energy, uint8_t *d_codes, int64_t *d_sweep, void *stream)
{
    const std::string name = "evc_sampler_best";
    if (!s) { set_error(name + ": null handle"); return 1; }
    if (!s->best_energy) { set_error(name + ": no record was started (evc_sampler_record_best)"); return 1; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const size_t n = (size_t)s->n_chains;
    EVC_CUDA(cudaSetDevice(s->device));
    if (d_energy) EVC_CUDA(cudaMemcpyAsync(d_energy, s->best_energy, n * sizeof(double), cudaMemcpyDeviceToDevice, st));
    if (d_codes) EVC_CUDA(cudaMemcpyAsync(d_codes, s->best_codes, n * s->L, cudaMemcpyDeviceToDevice, st));
    if (d_sweep) EVC_CUDA(cudaMemcpyAsync(d_sweep, s->best_sweep, n * sizeof(int64_t), cudaMemcpyDeviceToDevice, st));
    return 0;
}

int evc_sampler_descend(evc_sampler_t *s, int32_t sweeps, uint8_t *d_settled, int64_t *changes_out, void *stream)
{
    const std::string name = "evc_sampler_descend";
    if (!s) { set_error(name + ": null handle"); return 1; }
    if (sweeps < 0) { set_error(name + ": sweeps must be >= 0"); return 1; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    EVC_CUDA(cudaSetDevice(s->device));
    EVC_CUDA(cudaMemsetAsync(s->changes, 0, sizeof(unsigned long long), st));
    if (sweeps > 0) {
        const int rc = s->conditional ? descent_launch<true>(s, sweeps, d_settled, st)
                                      : descent_launch<false>(s, sweeps, d_settled, st);
        if (rc) return 1;
    }
    return read_changes(s, changes_out, st);
}

int evc_sampler_codes(const evc_sampler_t *s, uint8_t *d_codes_out, void *stream)
{
    if (!s || !d_codes_out) { set_error("evc_sampler_codes: null pointer"); return 1; }
    EVC_CUDA(cudaSetDevice(s->device));
    EVC_CUDA(cudaMemcpyAsync(d_codes_out, s->codes, (size_t)s->n_chains * s->L, cudaMemcpyDeviceToDevice,
                             reinterpret_cast<cudaStream_t>(stream)));
    return 0;
}

void evc_sampler_destroy(evc_sampler_t *s)
{
    if (!s) return;
    cudaSetDevice(s->device);
    sampler_free(s);
}

}  // extern "C"
