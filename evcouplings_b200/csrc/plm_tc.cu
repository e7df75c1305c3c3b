// Hot path (a) as dense one-hot contractions on the Hopper tensor cores (wgmma / TMA / mbarrier).
//
// The gather kernels (plm_gather.cu) compute the same objective and gradient without tensor cores;
// `bench.py --forward gather --backward gather` times them against this path.
//
// Maths.  With X[n,(j,b)] = [s_nj = b] (one-hot, exact in bf16), the couplings W[(i,a),(j,b)] = J_ij(a,b) and
// the residuals R[n,(i,a)] = r_ni(a):
//     forward   Zt[(i,a), n]     = sum_(j,b) W[(i,a),(j,b)] * X[n,(j,b)]          (logits without h)
//     backward  Gd[(j,b),(i,a)]  = sum_n     X[n,(j,b)]     * R[n,(i,a)]
//               g_J(i<j)[a][b]   = Gd[(j,b),(i,a)] + Gd[(i,a),(j,b)]
// Precision mode 0 (fp32-equivalent, default): the real-valued operand (W or R) is split in two bf16 terms
// (hi = rn(v), lo = rn(v - hi)): 16 mantissa bits, relative error 2^-17 per term; both products accumulate into the
// SAME fp32 register accumulator.  Precision mode 1 ("bf16 tiles", BASELINE configs[4]): hi only, one product per term.
//
// Operands:
//     forward : Wt_hi, Wt_lo [Mp][Kw] bf16 (written by expand_tc every evaluation; K-major TMA 2-D, SWIZZLE_128B),
//               X as a 2:4-sparse operand in fragment-ready form (build_xsp_kernel; static, or per sequence chunk)
//     backward: Xt [Mp][Kp] bf16 (static), Rt_hi, Rt_lo [Np][Kp] bf16 (written by plm_softmax_kernel), K-major
//               TMA 2-D, SWIZZLE_128B (the canonical wgmma shared-memory layout)
//
// tc_gemm_kernel<SINGLE> (backward): one CTA of 384 threads per 128 x 192 output tile, K blocks of 64.
//     warpgroup 0        TMA producer (one thread): shared-memory ring (3 x 64 KB / 5 x 40 KB depending on mode),
//                        mbarrier expect_tx; hands its registers to the consumers (setmaxnreg)
//     warpgroups 1, 2    consumers, 64 rows of the tile each: per K block 4 (x 2 in mode 0) wgmma.mma_async
//                        m64n192k16; one K block of wgmmas stays in flight while the stage before it is released
// The backward has few tiles (33 x 22 at L = 200) and long K (the sequences): its K extent is split into slices
// (backward_ksplit) so that the work units fill whole waves of the GPU; each slice writes its own plane of Gd and
// finalize_pairs_tc sums the planes in a fixed order.
//
// tc_sparse_logits_kernel<SINGLE> (forward): the one-hot X has at most 2 nonzeros in every aligned group of 4 K
// columns (a group touches at most two sites), so it is the 2:4-sparse A operand of wgmma.mma_async.sp, which issues
// half the multiply-adds of the dense instruction.  Sequences on M, states (i,a) on N: one CTA per 256 sequences x
// 192 states when K is one accumulation chain (L q <= 8192), else per 128 x 192; K blocks of 64 = two m64n192k32
// sparse steps (x 2 in mode 0: hi and lo share the A registers).  The CTAs that share a 192-row slice of Wt run in
// 2-CTA clusters: each loads half of every W stage and multicasts it.
// Both kernels: the tensor core's fp32 accumulation does not round to nearest, so a long accumulation chain picks up
// a systematic bias; at most k_chunk K blocks are accumulated by wgmma before the chunk is added into a second
// register accumulator with IEEE round-to-nearest adds, which keeps the result at the level of a plain fp32 sum.
#include <cuda.h>
#include <cuda_bf16.h>

#include <stdlib.h>

#include <algorithm>

#include "common.cuh"
#include "internal.h"

namespace evc {

constexpr int TC_BM = 128;
constexpr int TC_BN = 192;
constexpr int TC_BK = 64;
constexpr int TC_MAX_STAGES = 8;   // ring depth is chosen at launch from the stage size (hi+lo: 3-4, bf16x1: 5)
constexpr int TC_A_BYTES = TC_BM * TC_BK * 2;        // 16384
constexpr int TC_B_BYTES = TC_BN * TC_BK * 2;        // 24576
constexpr int TC_SMEM_LIMIT = 232448;                // 227 KB opt-in shared memory per CTA
constexpr int TC_SMEM_HEAD = 2048;                   // 1 KB alignment slack + 1 KB of mbarriers
constexpr int TC_THREADS = 384;   // warpgroup 0: TMA producer, warpgroups 1-2: wgmma consumers
constexpr int TC_CONSUMERS = 256; // consumer threads; each one releases a stage after its wgmma.wait_group
constexpr int TC_K_CHUNK = 32;    // K blocks (of 64) accumulated by wgmma before promotion to an fp32 add
constexpr int TC_MAX_KSPLIT = 8;  // K slices of the backward product (planes of Gd); the default picks 1-4
constexpr int TC_REG_PRODUCER = 40;
constexpr int TC_REG_CONSUMER = 232;                 // 128 x 40 + 256 x 232 <= 64 K registers per SM
constexpr int TC_REG_PRODUCER_PAIR = 24;             // the 256-row sparse forward: two accumulators per thread,
constexpr int TC_REG_CONSUMER_PAIR = 240;            // which spill at 232; 128 x 24 + 256 x 240 <= 64 K

// ---- PTX wrappers ---------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_wait_bounded(uint64_t *bar, uint32_t parity)
{
    // spin with a cap so that a programming error becomes a trap instead of a hung GPU
    uint32_t done = 0;
    for (uint64_t it = 0; it < (1ull << 31); it++) {
        asm volatile(
            "{\n.reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n}\n"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
        if (done) return;
    }
    __trap();
}

__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ void tma_load_2d(void *smem_dst, const CUtensorMap *tmap, int c0, int c1, uint64_t *bar)
{
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}

// same, with an L2 cache-policy hint (used to keep the operand that every tile re-reads resident in L2)
__device__ __forceinline__ void tma_load_2d_hint(void *smem_dst, const CUtensorMap *tmap, int c0, int c1,
                                                 uint64_t *bar, uint64_t policy)
{
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint "
        "[%0], [%1, {%3, %4}], [%2], %5;"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
        "l"(policy)
        : "memory");
}
__device__ __forceinline__ uint64_t l2_policy_evict_last()
{
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}

template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(N)); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// keeps the compiler from touching accumulator registers across the asynchronous wgmma window
template <int R>
__device__ __forceinline__ void fence_regs(float *d)
{
#pragma unroll
    for (int i = 0; i < R; i++) asm volatile("" : "+f"(d[i])::"memory");
}

// named barrier of the two consumer warpgroups (barrier 0 is __syncthreads)
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(TC_CONSUMERS) : "memory"); }

// K-major, 128-byte swizzle, densely packed 8-row x 128-byte atoms (SBO = 1024 B); sm_90 wgmma descriptor.
// Offsets inside the ring (16-byte units) are added to the start-address field; the operand tiles are 1024-byte
// aligned, and a 16-wide K slice is 32 bytes further along the swizzled row.
__device__ __forceinline__ uint64_t make_desc_sw128(const void *smem_ptr)
{
    const uint32_t addr = smem_u32(smem_ptr);
    uint64_t d = 0;
    d |= (uint64_t)((addr >> 4) & 0x3FFF);       // start address >> 4          bits [0,14)
    d |= (uint64_t)1 << 16;                      // leading byte offset (unused for swizzled K-major) bits [16,30)
    d |= (uint64_t)(1024 >> 4) << 32;            // stride byte offset >> 4      bits [32,46)
    d |= (uint64_t)1 << 62;                      // layout type SWIZZLE_128B    bits [62,64)
    return d;
}

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, bf16 operands from shared memory (both K-major), fp32 accumulator in
// registers.  Fragment of thread t of the warpgroup: d[4c + e] is row 16 (t / 32) + (t % 32) / 4 + 8 (e / 2),
// column 8 c + 2 (t % 4) + (e % 2).  scale_d == 0 overwrites the accumulator.
template <int N>
__device__ __forceinline__ void wgmma_bf16(float *d, uint64_t da, uint64_t db, uint32_t scale_d);
template <>
__device__ __forceinline__ void wgmma_bf16<192>(float *d, uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n.reg .pred p;\n"
        "setp.ne.b32 p, %98, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n192k16.f32.bf16.bf16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95"
        "}, %96, %97, p, 1, 1, 0, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
        : "l"(da), "l"(db), "r"(scale_d));
}
template <>
__device__ __forceinline__ void wgmma_bf16<176>(float *d, uint64_t da, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n.reg .pred p;\n"
        "setp.ne.b32 p, %90, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n176k16.f32.bf16.bf16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87"
        "}, %88, %89, p, 1, 1, 0, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87])
        : "l"(da), "l"(db), "r"(scale_d));
}

// D[64 x 192] (+)= A[64 x 32] * B[192 x 32]^T with A 2:4-sparse along K, from registers: a[0..3] hold the two kept
// values of groups (t % 4) and 4 + (t % 4) of rows r and r + 8 (r = 16 (t / 32) + (t % 32) / 4) in the order
// {r, g}, {r + 8, g}, {r, g + 4}, {r + 8, g + 4}; e holds their positions (build_xsp_kernel).  Sparsity selector 0.
__device__ __forceinline__ void wgmma_sp_bf16_192(float *d, const uint4 &a, uint32_t e, uint64_t db, uint32_t scale_d)
{
    asm volatile(
        "{\n.reg .pred p;\n"
        "setp.ne.b32 p, %102, 0;\n"
        "wgmma.mma_async.sp.sync.aligned.m64n192k32.f32.bf16.bf16 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95"
        "}, {%96, %97, %98, %99}, %100, %101, 0, p, 1, 1, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
        : "r"(a.x), "r"(a.y), "r"(a.z), "r"(a.w), "l"(db), "r"(e), "r"(scale_d));
}

__device__ __forceinline__ uint4 lds128(uint32_t addr)
{
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t addr)
{
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
// ---- cluster helpers (2-CTA clusters of the sparse forward) -----------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank()
{
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync()
{
    asm volatile("barrier.cluster.arrive.release;\nbarrier.cluster.wait.acquire;" ::: "memory");
}
// arrive on the mbarrier at the same shared-memory offset in CTA `rank` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t *bar, uint32_t rank)
{
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(rank));
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
// TMA 2-D load written to the same shared-memory offset of every CTA in `mask`, each of whose mbarrier at the
// offset of `bar` receives the bytes
__device__ __forceinline__ void tma_load_2d_multicast(void *smem_dst, const CUtensorMap *tmap, int c0, int c1,
                                                      uint64_t *bar, uint16_t mask, uint64_t policy)
{
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster.L2::cache_hint"
        " [%0], [%1, {%4, %5}], [%2], %3, %6;"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "h"(mask), "r"(c0),
        "r"(c1), "l"(policy)
        : "memory");
}

// one 64-wide K block: 4 slices of 16, each one wgmma (bf16 tiles) or two (hi + lo: A * B and A2 * B2)
template <int N>
__device__ __forceinline__ void wgmma_kblock(float *acc, uint64_t a, uint64_t b, uint64_t a2, uint64_t b2, bool two,
                                             bool overwrite)
{
#pragma unroll
    for (int k = 0; k < TC_BK / 16; k++) {
        const uint64_t koff = (uint64_t)((k * 16 * 2) >> 4);
        wgmma_bf16<N>(acc, a + koff, b + koff, (overwrite && k == 0) ? 0u : 1u);
        if (two) wgmma_bf16<N>(acc, a2 + koff, b2 + koff, 1u);
    }
}

// Consumer main loop over K blocks [kb0, kb1) of the ring: waits for each stage, issues its wgmmas, and releases a
// stage once the wgmma group that read it has completed (one group stays in flight).  Operand offsets are in
// 16-byte units from the start of a stage.  Returns with every wgmma complete.
template <int N>
__device__ __forceinline__ void tc_mainloop(float *acc, uint64_t *full, uint64_t *empty, int &s, uint32_t &ph,
                                            int n_stages, int stage_bytes, int kb0, int kb1, uint64_t desc0,
                                            uint64_t off_a, uint64_t off_b, uint64_t off_a2, uint64_t off_b2, bool two)
{
    int prev = -1;
    for (int kb = kb0; kb < kb1; kb++) {
        mbar_wait_bounded(&full[s], ph);
        wgmma_fence();
        const uint64_t d = desc0 + (uint64_t)((s * stage_bytes) >> 4);
        wgmma_kblock<N>(acc, d + off_a, d + off_b, d + off_a2, d + off_b2, two, kb == kb0);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0) mbar_arrive(&empty[prev]);
        prev = s;
        if (++s == n_stages) { s = 0; ph ^= 1u; }
    }
    wgmma_wait<0>();
    fence_regs<N / 2>(acc);
    if (prev >= 0) mbar_arrive(&empty[prev]);
}

// Tile enumeration: M tiles are swept in groups of `mgroup`; inside a group the M index is fastest, then the N
// tile.  The sparse forward passes its state tiles as M: a group whose slice of the coupling operand fits in L2
// (about 24 MB, see forward_group) stays resident while every sequence tile passes by; the backward uses one
// group (neighbouring CTAs share the operand tiles of the same K range).
__device__ __forceinline__ void decode_tile(int tile, int m_tiles, int n_tiles, int mgroup, int &m_tile, int &n_tile)
{
    const int full = (m_tiles / mgroup) * mgroup * n_tiles;
    if (tile < full) {
        const int per = mgroup * n_tiles;
        const int g = tile / per, r = tile - g * per;
        n_tile = r / mgroup;
        m_tile = g * mgroup + (r - n_tile * mgroup);
    } else {
        const int rem = m_tiles % mgroup, r = tile - full;
        n_tile = r / rem;
        m_tile = (m_tiles / mgroup) * mgroup + (r - n_tile * rem);
    }
}

// shared-memory layout of the tensor-core kernels: [mbarriers, 1 KB][operand ring, 1024-byte aligned]
struct TcSmem {
    uint64_t *full, *empty;
    unsigned char *ring;
};
__device__ __forceinline__ TcSmem tc_smem_layout(unsigned char *smem_dyn)
{
    unsigned char *base = reinterpret_cast<unsigned char *>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) &
                                                            ~static_cast<uintptr_t>(1023));
    TcSmem l;
    l.full = reinterpret_cast<uint64_t *>(base);
    l.empty = l.full + TC_MAX_STAGES;
    l.ring = base + 1024;
    return l;
}
__device__ __forceinline__ void tc_init_barriers(const TcSmem &l, int n_stages)
{
    if (threadIdx.x == 0) {
        for (int s = 0; s < n_stages; s++) {
            mbar_init(&l.full[s], 1);
            mbar_init(&l.empty[s], TC_CONSUMERS);
        }
        mbar_fence_init();
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------------------------------
// Backward GEMM, one 128 x 192 tile per CTA:
//     Gd[(j,b),(i,a)]  = sum_n Xt[(j,b), n] * (Rt_hi [+ Rt_lo])[(i,a), n]
// Stage layout (the optional lo operand is LAST so that the bf16x1 precision mode uses a compact prefix and
// a deeper ring): [A 16 KB][B_hi 24 KB][B_lo 24 KB].
// SINGLE (precision mode 1, "bf16 tiles"): the lo operand is neither loaded nor multiplied.
// Split K: the K blocks are cut into `ksplit` slices of ceil(num_kb / ksplit) blocks; CTA index =
// slice * tiles + tile (slice slowest: the CTAs of a wave stream the same K range through L2), and slice s writes
// its own output plane D + s * plane.  Every slice is non-empty (the host picks ksplit so).
// ACC (sequence chunks, see evc_plm_eval_data): slices below acc_planes add their sum to the plane
// (D += acc; every CTA owns its tile of its plane, so the chunks' products are added in chunk order without
// atomics); slices at or above acc_planes store as in the default mode (the plane is touched for the first time).
// ---------------------------------------------------------------------------------------------------
template <int SINGLE, int ACC = 0>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_gemm_kernel(const __grid_constant__ CUtensorMap tm0, const __grid_constant__ CUtensorMap tm1,
               const __grid_constant__ CUtensorMap tm2, float *__restrict__ D, int64_t ldd, int m_tiles, int n_tiles,
               int num_kb, int k_chunk, int mgroup, int n_stages, int ksplit, int64_t plane, int acc_planes)
{
    constexpr int BYTES0 = TC_A_BYTES;                              // operand 0: A (Xt), 128 rows
    constexpr int BYTES1 = TC_B_BYTES;                              // operand 1: B_hi, 192 rows
    constexpr int BYTES2 = TC_B_BYTES;                              // operand 2: B_lo, optional
    constexpr int stage_bytes = BYTES0 + BYTES1 + (SINGLE ? 0 : BYTES2);
    extern __shared__ unsigned char smem_dyn[];
    const TcSmem l = tc_smem_layout(smem_dyn);
    const int tiles = m_tiles * n_tiles;
    const int slice = (int)blockIdx.x / tiles;
    int m_tile, n_tile;
    decode_tile((int)blockIdx.x - slice * tiles, m_tiles, n_tiles, mgroup, m_tile, n_tile);
    const int kb_per = (num_kb + ksplit - 1) / ksplit;
    const int kb_begin = slice * kb_per, kb_end = min(num_kb, kb_begin + kb_per);
    tc_init_barriers(l, n_stages);

    if (threadIdx.x < 128) {
        // ===== TMA producer: one thread =====
        setmaxnreg_dec<TC_REG_PRODUCER>();
        if (threadIdx.x == 0) {
            int s = 0;
            uint32_t ph = 0;
            for (int kb = kb_begin; kb < kb_end; kb++) {
                mbar_wait_bounded(&l.empty[s], ph ^ 1u);
                unsigned char *st = l.ring + s * stage_bytes;
                mbar_expect_tx(&l.full[s], (uint32_t)stage_bytes);
                tma_load_2d(st, &tm0, kb * TC_BK, m_tile * TC_BM, &l.full[s]);
                tma_load_2d(st + BYTES0, &tm1, kb * TC_BK, n_tile * TC_BN, &l.full[s]);
                if (!SINGLE) tma_load_2d(st + BYTES0 + BYTES1, &tm2, kb * TC_BK, n_tile * TC_BN, &l.full[s]);
                if (++s == n_stages) { s = 0; ph ^= 1u; }
            }
        }
    } else {
        // ===== consumers: warpgroup cw owns rows 64 cw .. 64 cw + 63 of the tile =====
        setmaxnreg_inc<TC_REG_CONSUMER>();
        const int cw = (threadIdx.x >> 7) - 1;
        constexpr uint64_t OFF1 = (uint64_t)(BYTES0 >> 4), OFF2 = (uint64_t)((BYTES0 + BYTES1) >> 4);
        const uint64_t arow = (uint64_t)((cw * 64 * TC_BK * 2) >> 4);      // this warpgroup's 64 rows of an A tile
        const uint64_t desc0 = make_desc_sw128(l.ring);
        float acc[TC_BN / 2], sum[TC_BN / 2];
#pragma unroll
        for (int u = 0; u < TC_BN / 2; u++) acc[u] = 0.f;
        const int n_chunks = (kb_end - kb_begin + k_chunk - 1) / k_chunk;
        int s = 0;
        uint32_t ph = 0;
        for (int c = 0; c < n_chunks; c++) {
            const int kb0 = kb_begin + c * k_chunk, kb1 = min(kb_end, kb0 + k_chunk);
            tc_mainloop<TC_BN>(acc, l.full, l.empty, s, ph, n_stages, stage_bytes, kb0, kb1, desc0,
                               arow, OFF1, arow, OFF2, !SINGLE);                       // A * B_hi + A * B_lo
#pragma unroll
            for (int u = 0; u < TC_BN / 2; u++) sum[u] = (c == 0) ? acc[u] : sum[u] + acc[u];
        }
        const int t = threadIdx.x & 127;
        const int64_t row = (int64_t)m_tile * TC_BM + cw * 64 + (t >> 5) * 16 + ((t & 31) >> 2);
        float *out = D + slice * plane + row * ldd + (int64_t)n_tile * TC_BN + 2 * (t & 3);
        if (ACC && slice < acc_planes) {
#pragma unroll
            for (int c8 = 0; c8 < TC_BN / 8; c8++) {
                float2 *p0 = reinterpret_cast<float2 *>(out + 8 * c8);
                float2 *p1 = reinterpret_cast<float2 *>(out + 8 * ldd + 8 * c8);
                const float2 v0 = __ldcs(p0), v1 = __ldcs(p1);
                __stcs(p0, make_float2(v0.x + sum[4 * c8], v0.y + sum[4 * c8 + 1]));
                __stcs(p1, make_float2(v1.x + sum[4 * c8 + 2], v1.y + sum[4 * c8 + 3]));
            }
            return;
        }
#pragma unroll
        for (int c8 = 0; c8 < TC_BN / 8; c8++) {             // streaming stores: do not pollute L2
            __stcs(reinterpret_cast<float2 *>(out + 8 * c8), make_float2(sum[4 * c8], sum[4 * c8 + 1]));
            __stcs(reinterpret_cast<float2 *>(out + 8 * ldd + 8 * c8), make_float2(sum[4 * c8 + 2], sum[4 * c8 + 3]));
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// Sparse forward, one tile of 128 sequences x 192 states per CTA:
//     Zt[(i,a), n] = sum_(j,b) X[n,(j,b)] * (Wt_hi [+ Wt_lo])[(i,a),(j,b)]
// A = X (2:4-sparse, from registers), B = Wt: the coupling matrix is symmetric, so row (i,a) of Wt is the K-major
// B operand of state (i,a).  B rows run past Mp in the last state tile: TMA fills them with zeros and they are not
// stored.  Stage layout: [W_hi 24 KB][A fragments 10 KB][W_lo 24 KB (hi+lo mode only)].
// Fragment-ready one-hot operand (build_xsp_kernel): sequence tile T (128 rows) and K block kb own the
// XSP_KB_BYTES contiguous bytes at (T * num_kb + kb) * XSP_KB_BYTES, in the order [warpgroup 0, 1][k32 step 0, 1]
// of XSP_STEP_BYTES: [A: one uint4 per thread of the warpgroup][metadata: one uint32 per thread].
// Clusters of cs = 1 or 2 CTAs along the sequence tiles share the state tile: with cs = 2 each CTA loads one 96-row
// half of every W stage and multicasts it to both, and a stage is free only when the consumers of both CTAs have
// released it (empty barrier: one arrival per consumer warp of each CTA).  An odd number of sequence tiles leaves
// the last cluster's second CTA without a tile: it still loads and multiplies (A of tile 0) so that its peer gets
// its half of W, and stores nothing.
// Tile order: clusters enumerate (state tile, sequence-tile pair) with decode_tile, the state tiles in groups of
// `group` whose W slice stays in L2 while every sequence tile passes by.  Each output element is one CTA's whole
// accumulation chain in a fixed order, so neither the grouping nor the cluster size changes a bit.
// PAIR (K is one accumulation chain, num_kb <= k_chunk): a CTA computes 256 sequences x 192 states, the sequence
// tiles 2P and 2P + 1 of its pair P; stage [W_hi 24 KB][A of 2P 10 KB][A of 2P + 1 10 KB][W_lo 24 KB].  Warpgroup
// cw owns tile 2P + cw as two 64-row blocks, each with its own A registers and accumulator (the registers that
// hold the promoted sum otherwise), and both blocks multiply the same W stage: per product the SM takes in 68 KB
// for 256 sequences instead of 2 x 58 KB.  A tile 2P + 1 beyond the last one still receives its A bytes (those of
// tile 0) and is multiplied but not stored.  Every logit is the same chain of the same instructions on the same
// fragments and W tiles as without PAIR, so Zt does not change by a bit.
// ---------------------------------------------------------------------------------------------------
constexpr int XSP_STEP_BYTES = 2560;                       // 128 x 16 B A fragments + 128 x 4 B metadata
constexpr int XSP_KB_BYTES = 4 * XSP_STEP_BYTES;           // 2 warpgroups x 2 k32 steps = 10240
constexpr int SP_W_HALF = (TC_BN / 2) * TC_BK * 2;         // 96 rows of a W stage: one TMA box, 12288 bytes

template <int SINGLE, int PAIR>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_sparse_logits_kernel(const __grid_constant__ CUtensorMap tm_hi, const __grid_constant__ CUtensorMap tm_lo,
                        const unsigned char *__restrict__ xsp, float *__restrict__ Zt, int64_t ldz, int64_t rows_z,
                        int state_tiles, int seq_tiles, int seq_units, int num_kb, int k_chunk, int group,
                        int n_stages)
{
    constexpr int TILES = PAIR ? 2 : 1;               // 128-sequence tiles per CTA
    constexpr int OFF_A = TC_B_BYTES;
    constexpr int OFF_LO = TC_B_BYTES + TILES * XSP_KB_BYTES;
    constexpr int stage_bytes = OFF_LO + (SINGLE ? 0 : TC_B_BYTES);
    extern __shared__ unsigned char smem_dyn[];
    const TcSmem l = tc_smem_layout(smem_dyn);
    uint32_t cs;
    asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(cs));
    const uint32_t rank = cluster_ctarank();
    int n_tile, unit;
    decode_tile((int)(blockIdx.x / cs), state_tiles, seq_units, group, n_tile, unit);
    const int seq_tile0 = (unit * (int)cs + (int)rank) * TILES;      // first 128-sequence tile of this CTA
    if (threadIdx.x == 0) {
        for (int s = 0; s < n_stages; s++) {
            mbar_init(&l.full[s], 1);
            mbar_init(&l.empty[s], 8 * cs);           // 8 consumer warps per CTA of the cluster
        }
        mbar_fence_init();
    }
    cluster_sync();                                   // the peer's barriers exist before anything is multicast

    if (threadIdx.x < 128) {
        // ===== TMA producer: one thread; W is re-read by every sequence tile -> evict_last =====
        setmaxnreg_dec<PAIR ? TC_REG_PRODUCER_PAIR : TC_REG_PRODUCER>();
        if (threadIdx.x == 0) {
            const uint64_t keep = l2_policy_evict_last();
            const unsigned char *src[TILES];
#pragma unroll
            for (int i = 0; i < TILES; i++) {
                const int tile = seq_tile0 + i;
                src[i] = xsp + (int64_t)(tile >= seq_tiles ? 0 : tile) * num_kb * XSP_KB_BYTES;
            }
            const int row0 = n_tile * TC_BN;
            int s = 0;
            uint32_t ph = 0;
            for (int kb = 0; kb < num_kb; kb++) {
                mbar_wait_bounded(&l.empty[s], ph ^ 1u);
                unsigned char *st = l.ring + s * stage_bytes;
                mbar_expect_tx(&l.full[s], (uint32_t)stage_bytes);
#pragma unroll
                for (int i = 0; i < TILES; i++)
                    bulk_g2s(st + OFF_A + i * XSP_KB_BYTES, src[i] + (int64_t)kb * XSP_KB_BYTES, XSP_KB_BYTES,
                             &l.full[s]);
                if (cs == 1) {
                    for (int h = 0; h < 2; h++) {
                        tma_load_2d_hint(st + h * SP_W_HALF, &tm_hi, kb * TC_BK, row0 + h * (TC_BN / 2), &l.full[s], keep);
                        if (!SINGLE)
                            tma_load_2d_hint(st + OFF_LO + h * SP_W_HALF, &tm_lo, kb * TC_BK, row0 + h * (TC_BN / 2),
                                             &l.full[s], keep);
                    }
                } else {
                    const int h = (int)rank;
                    tma_load_2d_multicast(st + h * SP_W_HALF, &tm_hi, kb * TC_BK, row0 + h * (TC_BN / 2), &l.full[s],
                                          (uint16_t)0x3, keep);
                    if (!SINGLE)
                        tma_load_2d_multicast(st + OFF_LO + h * SP_W_HALF, &tm_lo, kb * TC_BK, row0 + h * (TC_BN / 2),
                                              &l.full[s], (uint16_t)0x3, keep);
                }
                if (++s == n_stages) { s = 0; ph ^= 1u; }
            }
        }
    } else {
        // ===== consumers: warpgroup cw owns sequences 64 cw .. 64 cw + 63 of the tile (PAIR: all of tile cw) =====
        setmaxnreg_inc<PAIR ? TC_REG_CONSUMER_PAIR : TC_REG_CONSUMER>();
        const int cw = (threadIdx.x >> 7) - 1;
        const int t = threadIdx.x & 127;
        const uint32_t a_addr = smem_u32(l.ring) + OFF_A + cw * (PAIR ? XSP_KB_BYTES : 2 * XSP_STEP_BYTES) + 16 * t;
        const uint32_t e_addr = a_addr + 2048 - 12 * t;
        const uint64_t desc0 = make_desc_sw128(l.ring);
        constexpr uint64_t DLO = (uint64_t)(OFF_LO >> 4), DK32 = (uint64_t)((32 * 2) >> 4);   // K 32..63: 64 B on
        auto release = [&](int st) {
            if ((threadIdx.x & 31) == 0) {
                mbar_arrive_cluster(&l.empty[st], 0);
                if (cs == 2) mbar_arrive_cluster(&l.empty[st], 1);
            }
        };
        // d[4 c8 + e]: sequence seq0 + 8 (e / 2), state st0 + 8 c8 + (e % 2); a warp's store covers 8 consecutive
        // sequences (one 32-byte sector) of 4 states.  v[b] holds rows 64 b .. 64 b + 63 from row rb of 128-sequence
        // tile `tile`.  The row blocks are stored together, so both accumulators drain at the same pace and share
        // one address per state.
        auto store = [&](const float *const *v, int nb, int tile, int rb) {
            if (tile >= seq_tiles) return;
            const int64_t seq0 = (int64_t)tile * TC_BM + rb + (t >> 5) * 16 + ((t & 31) >> 2);
            const int64_t st0 = (int64_t)n_tile * TC_BN + 2 * (t & 3);
            bool col[2][2];
#pragma unroll
            for (int b = 0; b < 2; b++)
#pragma unroll
                for (int h = 0; h < 2; h++) col[b][h] = b < nb && seq0 + 64 * b + 8 * h < ldz;
            const int64_t nrows = rows_z - st0;      // this thread's states st0 .. st0 + nrows - 1 are rows of Zt
            float *p = Zt + st0 * ldz + seq0;
#pragma unroll
            for (int c8 = 0; c8 < TC_BN / 8; c8++) {
#pragma unroll
                for (int e = 0; e < 4; e++)
#pragma unroll
                    for (int b = 0; b < 2; b++)
                        if (8 * c8 + (e & 1) < nrows && col[b][e >> 1])
                            __stcs(p + (e & 1) * ldz + 64 * b + 8 * (e >> 1), v[b][4 * c8 + e]);
                p += 8 * ldz;
            }
        };
        if (PAIR) {
            // row blocks 0 and 1 of tile seq_tile0 + cw: fragments [row block][k32 step] of its A block
            float acc0[TC_BN / 2], acc1[TC_BN / 2];
#pragma unroll
            for (int u = 0; u < TC_BN / 2; u++) acc0[u] = acc1[u] = 0.f;
            int s = 0;
            uint32_t ph = 0;
            for (int kb = 0; kb < num_kb; kb++) {
                mbar_wait_bounded(&l.full[s], ph);
                const uint32_t so = (uint32_t)(s * stage_bytes);
                const uint4 a00 = lds128(a_addr + so), a01 = lds128(a_addr + so + XSP_STEP_BYTES);
                const uint4 a10 = lds128(a_addr + so + 2 * XSP_STEP_BYTES), a11 = lds128(a_addr + so + 3 * XSP_STEP_BYTES);
                const uint32_t e00 = lds32(e_addr + so), e01 = lds32(e_addr + so + XSP_STEP_BYTES);
                const uint32_t e10 = lds32(e_addr + so + 2 * XSP_STEP_BYTES), e11 = lds32(e_addr + so + 3 * XSP_STEP_BYTES);
                wgmma_fence();
                const uint64_t d = desc0 + (uint64_t)((s * stage_bytes) >> 4);
                const uint32_t sc = kb == 0 ? 0u : 1u;
                // each accumulator sees the order of the 128-row kernel: hi, lo of step 0, then hi, lo of step 1
                wgmma_sp_bf16_192(acc0, a00, e00, d, sc);
                wgmma_sp_bf16_192(acc1, a10, e10, d, sc);
                if (!SINGLE) {
                    wgmma_sp_bf16_192(acc0, a00, e00, d + DLO, 1u);
                    wgmma_sp_bf16_192(acc1, a10, e10, d + DLO, 1u);
                }
                wgmma_sp_bf16_192(acc0, a01, e01, d + DK32, 1u);
                wgmma_sp_bf16_192(acc1, a11, e11, d + DK32, 1u);
                if (!SINGLE) {
                    wgmma_sp_bf16_192(acc0, a01, e01, d + DLO + DK32, 1u);
                    wgmma_sp_bf16_192(acc1, a11, e11, d + DLO + DK32, 1u);
                }
                wgmma_commit();
                wgmma_wait<0>();                      // the A registers are reloaded for the next K block
                release(s);
                if (++s == n_stages) { s = 0; ph ^= 1u; }
            }
            fence_regs<TC_BN / 2>(acc0);
            fence_regs<TC_BN / 2>(acc1);
            const float *v[2] = {acc0, acc1};
            store(v, 2, seq_tile0 + cw, 0);
        } else {
            float acc[TC_BN / 2], sum[TC_BN / 2];
#pragma unroll
            for (int u = 0; u < TC_BN / 2; u++) acc[u] = 0.f;
            const int n_chunks = (num_kb + k_chunk - 1) / k_chunk;
            int s = 0;
            uint32_t ph = 0;
            for (int c = 0; c < n_chunks; c++) {
                const int kb0 = c * k_chunk, kb1 = min(num_kb, kb0 + k_chunk);
                for (int kb = kb0; kb < kb1; kb++) {
                    mbar_wait_bounded(&l.full[s], ph);
                    const uint32_t so = (uint32_t)(s * stage_bytes);
                    const uint4 a0 = lds128(a_addr + so), a1 = lds128(a_addr + so + XSP_STEP_BYTES);
                    const uint32_t e0 = lds32(e_addr + so), e1 = lds32(e_addr + so + XSP_STEP_BYTES);
                    wgmma_fence();
                    const uint64_t d = desc0 + (uint64_t)((s * stage_bytes) >> 4);
                    wgmma_sp_bf16_192(acc, a0, e0, d, kb == kb0 ? 0u : 1u);
                    if (!SINGLE) wgmma_sp_bf16_192(acc, a0, e0, d + DLO, 1u);
                    wgmma_sp_bf16_192(acc, a1, e1, d + DK32, 1u);
                    if (!SINGLE) wgmma_sp_bf16_192(acc, a1, e1, d + DLO + DK32, 1u);
                    wgmma_commit();
                    // the tensor core reads the A registers while the wgmmas run, and the next K block loads new
                    // ones: all of this block's wgmmas retire first (the other consumer warpgroup keeps the tensor
                    // cores busy)
                    wgmma_wait<0>();
                    release(s);
                    if (++s == n_stages) { s = 0; ph ^= 1u; }
                }
                fence_regs<TC_BN / 2>(acc);
#pragma unroll
                for (int u = 0; u < TC_BN / 2; u++) sum[u] = (c == 0) ? acc[u] : sum[u] + acc[u];
            }
            const float *v[2] = {sum, sum};
            store(v, 1, seq_tile0, cw * 64);
        }
    }
    cluster_sync();      // no CTA exits while its peer may still multicast into it or arrive on its barriers
}

// Fragment-ready 2:4 form of X[r][(j,b)] = [s_(n0+r),j = b] for the rows r < Xrows (exact zeros for r >= nreal and
// for the K padding (j,b) >= L q).  Per aligned group of 4 K columns (at most 2 nonzeros, see DESIGN.md) the kept
// positions i0 < i1 are the nonzeros, padded with zero positions: none -> (0, 1); one at p -> (0, 1) if p <= 1, else
// (0, p); two -> both.  Metadata nibble i0 | i1 << 2; kept values bf16 1.0 or 0.
// One thread per consumer thread t of a (sequence tile, K block, warpgroup, k32 step) fragment (layout at
// tc_sparse_logits_kernel): rows r = 64-row block + 16 (t / 32) + (t % 32) / 4 and r + 8; A words: groups t % 4 and
// 4 + t % 4 of both rows; metadata: groups 4 (t % 2) .. 4 (t % 2) + 3, row r in bits 0-15, row r + 8 in 16-31.
__device__ __forceinline__ uint32_t xsp_group(const uint32_t *__restrict__ msa4, int64_t Nld, int64_t n, bool real,
                                              int k, int lq, int q, uint32_t &vals)
{
    uint32_t mask = 0;
    if (real) {
#pragma unroll
        for (int p = 0; p < 4; p++) {
            const int kk = k + p;
            if (kk >= lq) break;
            const int j = kk / q, b = kk - j * q;
            const int code = (int)((msa4[(int64_t)(j >> 2) * Nld + n] >> (8 * (j & 3))) & 0xffu);
            mask |= (uint32_t)(code == b) << p;
        }
    }
    int i0 = 0, i1 = 1;
    if (__popc(mask) == 2) { i0 = __ffs(mask) - 1; i1 = 31 - __clz(mask); }
    else if (mask > 2) i1 = __ffs(mask) - 1;                      // one nonzero at 2 or 3
    vals = (((mask >> i0) & 1u) ? 0x3F80u : 0u) | ((((mask >> i1) & 1u) ? 0x3F80u : 0u) << 16);
    return (uint32_t)(i0 | (i1 << 2));
}

__global__ void build_xsp_kernel(const uint32_t *__restrict__ msa4, unsigned char *__restrict__ out, int64_t n0,
                                 int64_t nreal, int64_t Nld, int L, int q, int num_kb, int64_t n_frag)
{
    const int64_t gt = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gt >= n_frag * 128) return;
    const int64_t ci = gt >> 7;                       // fragment: ((T * num_kb + kb) * 2 + cw) * 2 + step
    const int t = (int)(gt & 127);
    const int step = (int)(ci & 1), cw = (int)((ci >> 1) & 1);
    const int64_t tkb = ci >> 2;
    const int kb = (int)(tkb % num_kb);
    const int64_t T = tkb / num_kb;
    const int64_t r0 = T * TC_BM + cw * 64 + (t >> 5) * 16 + ((t & 31) >> 2), r1 = r0 + 8;
    const int k0 = kb * TC_BK + step * 32, lq = L * q;
    const int c = t & 3, h = c & 1;
    uint32_t e = 0, v[2][2], unused;
#pragma unroll
    for (int rr = 0; rr < 2; rr++) {
        const int64_t r = rr ? r1 : r0;
#pragma unroll
        for (int i = 0; i < 4; i++)
            e |= xsp_group(msa4, Nld, n0 + r, r < nreal, k0 + 4 * (4 * h + i), lq, q, unused) << (16 * rr + 4 * i);
#pragma unroll
        for (int u = 0; u < 2; u++) xsp_group(msa4, Nld, n0 + r, r < nreal, k0 + 4 * (4 * u + c), lq, q, v[rr][u]);
    }
    unsigned char *frag = out + ci * XSP_STEP_BYTES;
    reinterpret_cast<uint4 *>(frag)[t] = make_uint4(v[0][0], v[1][0], v[0][1], v[1][1]);
    reinterpret_cast<uint32_t *>(frag + 2048)[t] = e;
}

// ---------------------------------------------------------------------------------------------------
// Fused forward: logits GEMM with the softmax / residual epilogue on the accumulator.
//   D[n, (i,a)] = sum_(j,b) X[n,(j,b)] * (Wp_hi + Wp_lo)[(i,a),(j,b)]        sequences on M
// An N tile is 8 sites in two halves of 4 x 21 + 4 zero columns (wgmma N = 176).  The accumulator goes through
// shared memory (the drained operand ring) so that each of the 256 consumer threads owns one sequence x 4 sites
// and sees whole 21-state logit vectors: +h, softmax, fx, residuals, bf16 hi/lo split written transposed
// (sequence fastest) straight into the operand of the backward GEMM.  The logits matrix never exists in HBM.
// Per-(site, 32-sequence group) partials of g_h / fx keep the reduction deterministic.  The whole K extent is one
// accumulation chain (the caller restricts the fused path to L*q <= 8192).
// ---------------------------------------------------------------------------------------------------
constexpr int TF_BN = 176;                         // 8 sites x 21 states + 8 pad
constexpr int TF_SITES = 8;
constexpr int TF_B_BYTES = TF_BN * TC_BK * 2;      // 22528
constexpr int TF_PITCH = TF_BN + 1;                // staging row pitch in floats (odd: conflict-free row reads)

template <int SINGLE>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_fwd_fused_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_whi,
                    const __grid_constant__ CUtensorMap tm_wlo, const float *__restrict__ h,
                    const uint32_t *__restrict__ msa4, const float *__restrict__ wts,
                    __nv_bfloat16 *__restrict__ Rt_hi, __nv_bfloat16 *__restrict__ Rt_lo, int64_t Kp,
                    float *__restrict__ gh_part, double *__restrict__ fx_part, PlmGeom g, int m_tiles, int n_tiles,
                    int num_kb, int n_stages)
{
    constexpr int Q = 21;                          // states per site of this instantiation (q = 21 or 20 -> S = 21)
    extern __shared__ unsigned char smem_dyn[];
    const TcSmem l = tc_smem_layout(smem_dyn);     // operand ring: [X 16 KB][W_hi 22 KB][W_lo 22 KB (hi+lo mode only)]
    constexpr int stage_bytes = TC_A_BYTES + TF_B_BYTES + (SINGLE ? 0 : TF_B_BYTES);
    // tiles enumerated with the site tile fastest => neighbouring CTAs share X tiles
    const int n_tile = blockIdx.x % n_tiles, m_tile = blockIdx.x / n_tiles;
    const int q = g.q;                             // 21, or 20 with the ignored gap (column 20 of a site is then zero)
    tc_init_barriers(l, n_stages);

    if (threadIdx.x < 128) {
        // ===== TMA producer =====
        setmaxnreg_dec<TC_REG_PRODUCER>();
        if (threadIdx.x == 0) {
            const uint64_t keep = l2_policy_evict_last();
            int s = 0;
            uint32_t ph = 0;
            for (int kb = 0; kb < num_kb; kb++) {
                mbar_wait_bounded(&l.empty[s], ph ^ 1u);
                unsigned char *st = l.ring + s * stage_bytes;
                mbar_expect_tx(&l.full[s], (uint32_t)stage_bytes);
                tma_load_2d(st, &tm_x, kb * TC_BK, m_tile * TC_BM, &l.full[s]);
                tma_load_2d_hint(st + TC_A_BYTES, &tm_whi, kb * TC_BK, n_tile * TF_BN, &l.full[s], keep);
                if (!SINGLE)
                    tma_load_2d_hint(st + TC_A_BYTES + TF_B_BYTES, &tm_wlo, kb * TC_BK, n_tile * TF_BN, &l.full[s], keep);
                if (++s == n_stages) { s = 0; ph ^= 1u; }
            }
        }
        return;
    }
    setmaxnreg_inc<TC_REG_CONSUMER>();
    const int ct = threadIdx.x - 128;              // consumer thread 0..255
    {
        // ===== logits: warpgroup cw owns sequences 64 cw .. 64 cw + 63 of the tile =====
        const int cw = ct >> 7;
        const uint64_t arow = (uint64_t)((cw * 64 * TC_BK * 2) >> 4);
        constexpr uint64_t OFFH = (uint64_t)(TC_A_BYTES >> 4), OFFL = (uint64_t)((TC_A_BYTES + TF_B_BYTES) >> 4);
        float acc[TF_BN / 2];
#pragma unroll
        for (int u = 0; u < TF_BN / 2; u++) acc[u] = 0.f;
        int s = 0;
        uint32_t ph = 0;
        tc_mainloop<TF_BN>(acc, l.full, l.empty, s, ph, n_stages, stage_bytes, 0, num_kb, make_desc_sw128(l.ring),
                           arow, OFFH, arow, OFFL, !SINGLE);
        // every TMA load of this tile has landed and both warpgroups are done reading: the ring becomes staging
        consumer_sync();
        float *stg = reinterpret_cast<float *>(l.ring);
        const int t = ct & 127;
        const int r0 = cw * 64 + (t >> 5) * 16 + ((t & 31) >> 2);
#pragma unroll
        for (int c8 = 0; c8 < TF_BN / 8; c8++) {
            const int col = 8 * c8 + 2 * (t & 3);
            stg[r0 * TF_PITCH + col] = acc[4 * c8];
            stg[r0 * TF_PITCH + col + 1] = acc[4 * c8 + 1];
            stg[(r0 + 8) * TF_PITCH + col] = acc[4 * c8 + 2];
            stg[(r0 + 8) * TF_PITCH + col + 1] = acc[4 * c8 + 3];
        }
        consumer_sync();
    }
    // ===== fused epilogue: thread = sequence, 4 sites =====
    const float *stg = reinterpret_cast<const float *>(l.ring);
    const int ehalf = ct >> 7;                    // which 4 sites of the tile's 8
    const int r = ct & 127;                       // sequence within the tile
    const int quad = r >> 5, lane = r & 31;
    const int ntile_part = m_tiles * 4;           // partial slots per site: (sequence tile, 32-sequence group)
    const int64_t n = (int64_t)m_tile * TC_BM + r;
    const int64_t nc = n < g.N ? n : g.N - 1;
    const float wn = n < g.N ? wts[nc] : 0.f;
    const float *v = stg + r * TF_PITCH + ehalf * 88;
#pragma unroll
    for (int s = 0; s < 4; s++) {
        const int i = n_tile * TF_SITES + ehalf * 4 + s;
        if (i >= g.L) break;                                   // padding sites of the last tile (uniform)
        const int si = (int)((msa4[(int64_t)(i >> 2) * g.Nld + nc] >> (8 * (i & 3))) & 0xffu);
        const float w = si < q ? wn : 0.f;
        float z[Q];
        float mx = -INFINITY;
#pragma unroll
        for (int a = 0; a < Q; a++) {
            z[a] = (a < q) ? v[s * Q + a] + h[i * q + a] : -INFINITY;
            mx = fmaxf(mx, z[a]);
        }
        float zs = 0.f, sum = 0.f;
#pragma unroll
        for (int a = 0; a < Q; a++) {
            if (a == si) zs = z[a];
            z[a] = (a < q) ? expf(z[a] - mx) : 0.f;
            sum += z[a];
        }
        const double fx_local = (w == 0.f) ? 0.0 : -((double)w * (double)(zs - mx - logf(sum)));
        const float inv = w / sum;
        float *ghp = gh_part + ((int64_t)i * ntile_part + m_tile * 4 + quad) * g.S;
#pragma unroll
        for (int a = 0; a < Q; a++) {
            const float rr = z[a] * inv - (a == si ? w : 0.f);
            if (a < q) {
                if (n < g.N) {
                    const int64_t off = ((int64_t)i * q + a) * Kp + n;
                    const __nv_bfloat16 hi = __float2bfloat16_rn(rr);
                    Rt_hi[off] = hi;
                    if (!SINGLE) Rt_lo[off] = __float2bfloat16_rn(rr - __bfloat162float(hi));
                }
            }
            const float tot = warp_sum(rr);
            if (lane == 0) ghp[a] = (a < q) ? tot : 0.f;
        }
        const double fw = warp_sum(fx_local);
        if (lane == 0) fx_part[(int64_t)i * ntile_part + m_tile * 4 + quad] = fw;
    }
}

// ---- expand: Wt[(i,a)][(j,b)] = J_ij(a,b) (i < j) and J_ji(b,a) (i > j) as bf16 hi + lo ------------------
// One CTA per pair of site tiles (I, J), I <= J, of EXP_SITES sites each.  The J_ij blocks with i in I, j in J,
// i < j are read once into shared memory (for one i they are contiguous in x), then the (I, J) and the (J, I)
// tiles of the operand are written row by row: each row of a tile is EXP_SITES * q contiguous K indices, stored
// as bf16x2.  The diagonal blocks (i = j) of the operand stay zero.  hi = rn(v), lo = rn(v - hi) per element.
// PADDED: rows of the fused forward's operand, regrouped as [site tile][8 sites x q states (+ zero pad to 176)].
constexpr int EXP_SITES = 4;
constexpr int EXP_THREADS = 256;

template <bool PADDED>
__device__ __forceinline__ int64_t expand_row(int i, int a, int q)
{
    // padded row base of a site: tile of 8 sites = two halves of 88 rows (4 sites x 21 states + 4 zero rows)
    if (PADDED) return (int64_t)(i / TF_SITES) * TF_BN + ((i % TF_SITES) / 4) * 88 + (i % 4) * 21 + a;
    return (int64_t)i * q + a;
}

// 4-byte global -> shared asynchronous copy (many loads in flight without holding registers)
__device__ __forceinline__ void cp_async4(void *smem_dst, const void *gmem_src)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// WIDE (q > 21): the blocks live in dynamic shared memory of exp_wide_smem(q) bytes (64 KB at q = 32, with the
// opt-in attribute); q <= 21 keeps the 28 KB static array.
constexpr int EXP_STATIC_Q = 21;
static size_t exp_wide_smem(int q) { return (size_t)EXP_SITES * EXP_SITES * q * q * sizeof(float); }

template <bool PADDED, bool WIDE = false>
__global__ void __launch_bounds__(EXP_THREADS)
expand_tc_kernel(const float *__restrict__ x, __nv_bfloat16 *__restrict__ W_hi, __nv_bfloat16 *__restrict__ W_lo,
                 int L, int q, int64_t ldw, int single)
{
    __shared__ float sJ_static[WIDE ? 1 : EXP_SITES * EXP_SITES * EXP_STATIC_Q * EXP_STATIC_Q];
    extern __shared__ float sJ_dyn[];
    float *const sJ = WIDE ? sJ_dyn : sJ_static;            // [i - i0][j - j0][a][b], blocks of q * q
    const int ti = blockIdx.y, tj = blockIdx.x;
    if (tj < ti) return;
    const int i0 = ti * EXP_SITES, j0 = tj * EXP_SITES;
    const int ni = min(EXP_SITES, L - i0), nj = min(EXP_SITES, L - j0);
    const int qq = q * q;
    for (int ii = 0; ii < ni; ii++) {
        const int i = i0 + ii, jlo = max(j0, i + 1);
        if (jlo >= j0 + nj) continue;
        const float *src = x + (int64_t)L * q + ((int64_t)i * (2 * L - i - 1) / 2 + (jlo - i - 1)) * qq;
        float *dst = sJ + (ii * EXP_SITES + (jlo - j0)) * qq;
        const int n = (j0 + nj - jlo) * qq;
        for (int e = threadIdx.x; e < n; e += blockDim.x) cp_async4(dst + e, src + e);
    }
    cp_async_wait_all();
    __syncthreads();
    // Tile with row sites [r0, r0 + nr) and K sites [c0, c0 + nc): one warp per row, lane l owns the K index pairs
    // (2 l, 2 l + 1) and (2 l + 64, 2 l + 65) of the row (a row has at most 4 * q <= 128 = 4 * 32).  The element at row
    // (r, ra), K index (c, cb) is J_rc(ra, cb) for r < c, J_cr(cb, ra) for r > c and 0 for r = c; with local site
    // indices rs = r - r0, cs = c - c0 its place in sJ is rowN + colN (r < c, then r0 = i0, c0 = j0) or
    // rowT + colT (r > c, then c0 = i0, and r0 = j0 or r0 = i0 = j0).  The row offset c0 * q is even (c0 = 4 t).
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    auto write_tile = [&](int r0, int nr, int c0, int nc) {
        const int width = nc * q;
        int csite[4], colN[4], colT[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int c = 2 * lane + 64 * (k >> 1) + (k & 1);
            const int cs = c / q, cb = c - cs * q;
            csite[k] = c0 + cs;
            colN[k] = cs * qq + cb;
            colT[k] = cs * EXP_SITES * qq + cb * q;
        }
        for (int rr = warp; rr < nr * q; rr += EXP_THREADS / 32) {
            const int rs = rr / q, ra = rr - rs * q, r = r0 + rs;
            const int rowN = rs * EXP_SITES * qq + ra * q, rowT = rs * qq + ra;
            const int64_t off = expand_row<PADDED>(r, ra, q) * ldw + (int64_t)c0 * q;
            auto elem = [&](int k) -> float {
                if (r < csite[k]) return sJ[rowN + colN[k]];
                if (r > csite[k]) return sJ[rowT + colT[k]];
                return 0.f;
            };
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int c = 2 * lane + 64 * h;
                if (c >= width) continue;
                const float v0 = elem(2 * h);
                const __nv_bfloat16 h0 = __float2bfloat16_rn(v0);
                const __nv_bfloat16 l0 = __float2bfloat16_rn(v0 - __bfloat162float(h0));
                if (c + 1 < width) {
                    const float v1 = elem(2 * h + 1);
                    const __nv_bfloat16 h1 = __float2bfloat16_rn(v1);
                    const __nv_bfloat16 l1 = __float2bfloat16_rn(v1 - __bfloat162float(h1));
                    *reinterpret_cast<__nv_bfloat162 *>(W_hi + off + c) = __halves2bfloat162(h0, h1);
                    if (!single) *reinterpret_cast<__nv_bfloat162 *>(W_lo + off + c) = __halves2bfloat162(l0, l1);
                } else {
                    W_hi[off + c] = h0;
                    if (!single) W_lo[off + c] = l0;
                }
            }
        }
    };
    write_tile(i0, ni, j0, nj);
    if (ti != tj) write_tile(j0, nj, i0, ni);
}

// one-hot operand of the forward product: X[r][(j,b)], K = (j,b) fastest, for the sequences n0 + r of a chunk.
// One CTA per row of the buffer: rows r >= nreal (beyond the chunk's last real sequence) are written as exact zeros,
// so a buffer that still holds the previous chunk is fully overwritten.  The K padding (j,b) >= L q is never
// written (zeroed once at allocation).
__global__ void build_x_kernel(const uint32_t *__restrict__ msa4, __nv_bfloat16 *__restrict__ X, int64_t n0,
                               int64_t nreal, int64_t Nld, int L, int q, int64_t ldx)
{
    const int64_t r = blockIdx.x;
    const bool real = r < nreal;
    for (int e = threadIdx.x; e < L * q; e += blockDim.x) {
        const int j = e / q, b = e - j * q;
        const int code = real ? (int)((msa4[(int64_t)(j >> 2) * Nld + n0 + r] >> (8 * (j & 3))) & 0xffu) : 255;
        X[r * ldx + e] = __float2bfloat16(code == b ? 1.0f : 0.0f);
    }
}

// softmax + residuals from the logits Zt[(i,a)][n]: thread = two adjacent sequences (8-byte loads of the
// logits, 4-byte bf16x2 stores of the residuals), CTA = 128 threads = 256 sequences of one site.
// ONEHOT = true: the "residual" is w_n [s_ni = a] (no logits read) -- the operand of the weighted pair counts
// f_ij = sum_n w_n [s_ni = a][s_nj = b] computed by the same tensor-core backward product (row a6).
// Sequence chunks: the CTAs cover the sequences n_base + [0, 256 gridDim.x) of a chunk (n_base is a multiple of
// 256).  Zt is read and Rt written at chunk-local columns; msa4 and wts are read at global sequence indices; the
// g_h / fx partials go to the global tile n_base / 256 + blockIdx.x of arrays sized for the whole shard (stride
// ntiles), so that plm_finalize_fields_n sums them in the same order whatever the chunking.
// RUNTIME_Q: Q is a register bound (8, 16 or 32) and the kernel serves every q = g.q <= Q; the states q..Q-1 of the
// registers take no part (logit -inf, probability and residual 0, nothing read or written).  Otherwise q = Q.
template <int Q, bool ONEHOT, bool RUNTIME_Q = false>
__global__ void __launch_bounds__(128)
plm_softmax_kernel(const float *__restrict__ Zt, int64_t ldz, const float *__restrict__ h,
                   const uint32_t *__restrict__ msa4, const float *__restrict__ wts,
                   __nv_bfloat16 *__restrict__ Rt_hi, __nv_bfloat16 *__restrict__ Rt_lo, int64_t Kp,
                   float *__restrict__ gh_part, double *__restrict__ fx_part, PlmGeom g, int ntiles, int64_t n_base)
{
    static_assert(Q <= 32, "s_gh holds 32 states per warp");
    const int q = RUNTIME_Q ? g.q : Q;
    __shared__ float s_gh[4 * 32];
    __shared__ double s_fx[4];
    const int tile = (int)(n_base >> 8) + blockIdx.x, i = blockIdx.y;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t N = g.N;
    const int64_t nl = (int64_t)blockIdx.x * 256 + 2 * tid;      // chunk-local column
    const int64_t n0 = n_base + nl;                                // global sequence
    // clamped, even load position (rows of Zt / msa4 are padded beyond N, see plm_tcf_geometry / plm_pack_msa);
    // n_base is even and < N, so the clamped position stays inside the chunk
    const int64_t m0 = n0 < N ? n0 : ((N - 1) & ~(int64_t)1);
    const int64_t ml = m0 - n_base;
    const uint2 wi = *reinterpret_cast<const uint2 *>(msa4 + (int64_t)(i >> 2) * g.Nld + m0);
    const int sh = 8 * (i & 3);
    const int si[2] = {(int)((wi.x >> sh) & 0xffu), (int)((wi.y >> sh) & 0xffu)};
    float w[2];
    w[0] = (n0 < N && si[0] < q) ? wts[n0] : 0.f;
    w[1] = (n0 + 1 < N && si[1] < q) ? wts[n0 + 1] : 0.f;
    float z[2][Q];
    double fx_local = 0.0;
    if (ONEHOT) {
#pragma unroll
        for (int k = 0; k < 2; k++)
#pragma unroll
            for (int a = 0; a < Q; a++) z[k][a] = (a == si[k]) ? w[k] : 0.f;     // si >= q has w = 0
    } else {
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int a = 0; a < Q; a++) {
            if (a < q) {
                const float2 v = *reinterpret_cast<const float2 *>(Zt + ((int64_t)i * q + a) * ldz + ml);
                const float ha = h[i * q + a];
                z[0][a] = v.x + ha;
                z[1][a] = v.y + ha;
                mx[0] = fmaxf(mx[0], z[0][a]);
                mx[1] = fmaxf(mx[1], z[1][a]);
            } else {
                z[0][a] = -INFINITY;
                z[1][a] = -INFINITY;
            }
        }
#pragma unroll
        for (int k = 0; k < 2; k++) {
            float zs = 0.f, sum = 0.f;
#pragma unroll
            for (int a = 0; a < Q; a++) {
                if (a == si[k]) zs = z[k][a];
                z[k][a] = a < q ? expf(z[k][a] - mx[k]) : 0.f;
                sum += z[k][a];
            }
            if (w[k] != 0.f) fx_local -= (double)w[k] * (double)(zs - mx[k] - logf(sum));
            const float inv = w[k] / sum;
#pragma unroll
            for (int a = 0; a < Q; a++) z[k][a] = z[k][a] * inv - (a == si[k] ? w[k] : 0.f);
        }
    }
#pragma unroll
    for (int a = 0; a < Q; a++) {
        if (a >= q) break;                          // uniform over the CTA (RUNTIME_Q only)
        if (n0 < N) {
            // nl is even and Kp is a multiple of 64: the pair (nl, nl + 1) is 4-byte aligned and inside the row;
            // a sequence beyond N has weight 0, i.e. writes an exact zero into the K padding.  Columns of the last
            // chunk beyond N that this kernel does not write keep residuals of the previous chunk: finite values
            // (|r| <= w) that only ever meet the exact-zero columns build_xt_kernel writes for sequences >= N, so
            // they add exact zeros to the backward product.
            const int64_t off = ((int64_t)i * q + a) * Kp + nl;
            const __nv_bfloat162 hi = __floats2bfloat162_rn(z[0][a], z[1][a]);
            *reinterpret_cast<__nv_bfloat162 *>(Rt_hi + off) = hi;
            if (Rt_lo != nullptr)
                *reinterpret_cast<__nv_bfloat162 *>(Rt_lo + off) =
                    __floats2bfloat162_rn(z[0][a] - __low2float(hi), z[1][a] - __high2float(hi));
        }
        const float v = warp_sum(z[0][a] + z[1][a]);
        if (lane == 0) s_gh[warp * 32 + a] = v;
    }
    const double fw = warp_sum(fx_local);
    if (lane == 0) s_fx[warp] = fw;
    __syncthreads();
    if (tid < g.S) {                                // S <= 33 < 128 threads
        float tot = 0.f;
        if (tid < q)
            for (int ww = 0; ww < 4; ww++) tot += s_gh[ww * 32 + tid];
        gh_part[((int64_t)i * ntiles + tile) * g.S + tid] = tot;
    }
    if (tid == 0) fx_part[(int64_t)i * ntiles + tile] = (s_fx[0] + s_fx[1]) + (s_fx[2] + s_fx[3]);
}

// ---- one-hot operand (static per MSA, or rebuilt for every sequence chunk) ----------------------------------
// Column n of the buffer is sequence n0 + n; every column is written, as exact zeros for sequences >= N.
__global__ void build_xt_kernel(const uint32_t *__restrict__ msa4, __nv_bfloat16 *__restrict__ Xt, int64_t n0,
                                int64_t N, int64_t Nld, int64_t Kp, int L, int q)
{
    const int64_t n = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int j = blockIdx.y;
    if (n >= Kp) return;
    int code = 255;
    if (n0 + n < N) code = (int)((msa4[(int64_t)(j >> 2) * Nld + n0 + n] >> (8 * (j & 3))) & 0xffu);
    for (int b = 0; b < q; b++)
        Xt[((int64_t)j * q + b) * Kp + n] = __float2bfloat16(code == b ? 1.0f : 0.0f);
}

// g_J(i<j)[a][b] = scale * (Gd[(j,b),(i,a)] + Gd[(i,a),(j,b)]), Gd = plane 0 + plane 1 + ... (planes of the split-K
// backward, summed in this fixed order: deterministic).  One CTA per pair of site tiles (I, J), I <= J, of
// FIN_SITES sites: the (I, J) and (J, I) tiles of Gd are read row by row (FIN_SITES * q contiguous floats) into
// shared memory, then the gradient blocks of the tile are written in gJ order (for one i, the blocks j are
// contiguous).
constexpr int FIN_SITES = 4;
constexpr int FIN_W = FIN_SITES * 21;
constexpr int FIN_PITCH = FIN_W + 1;      // odd row pitch: the transposed reads are conflict-free
constexpr int FIN_THREADS = 256;
constexpr int FIN_SMEM = 2 * FIN_W * FIN_PITCH * (int)sizeof(float);    // 55.8 KB: four CTAs per SM
constexpr int FIN_BATCH = 8;              // row segments loaded per thread before they are stored
// WIDE (q > 21): the tile is FIN_SITES * q wide, row pitch wide_pitch = 4 q + 1 (odd), 132 KB at q = 32
static int fin_pitch(int q) { return q <= 21 ? FIN_PITCH : FIN_SITES * q + 1; }
static int fin_smem_bytes(int q) { return q <= 21 ? FIN_SMEM : 2 * (fin_pitch(q) - 1) * fin_pitch(q) * (int)sizeof(float); }

template <bool WIDE = false>
__global__ void __launch_bounds__(FIN_THREADS)
finalize_pairs_tc_kernel(const float *__restrict__ Gd, int planes, int64_t plane, float *__restrict__ gJ, int L,
                         int q, int Np, float scale, int wide_pitch)
{
    const int pitch = WIDE ? wide_pitch : FIN_PITCH;
    extern __shared__ float fin_smem[];
    float *sA = fin_smem;                     // sA[r][c] = Gd[(i0 q + r), (j0 q + c)]
    float *sB = fin_smem + (pitch - 1) * pitch; // sB[r][c] = Gd[(j0 q + r), (i0 q + c)]
    const int ti = blockIdx.y, tj = blockIdx.x;
    if (tj < ti) return;
    const int i0 = ti * FIN_SITES, j0 = tj * FIN_SITES;
    const int wi = min(FIN_SITES, L - i0) * q, wj = min(FIN_SITES, L - j0) * q;
    // rows of `cols` contiguous floats, the planes summed in order; FIN_BATCH vectors per thread in flight.  The
    // tile's first column col0 = 4 t q is a multiple of 4: float4 loads whenever the row length is one too.  A
    // thread's (row, vector) position advances by blockDim.x vectors per step (no division in the loop).
    auto stage = [&](float *dst, int row0, int rows, int col0, int cols) {
        const int V = (cols % 4 == 0) ? 4 : 1;
        const int nv = cols / V;
        const int dr = FIN_THREADS / nv, dc = FIN_THREADS - dr * nv;
        int r = threadIdx.x / nv, c = threadIdx.x - r * nv;
        while (r < rows) {
            float4 v[FIN_BATCH];
            int off[FIN_BATCH];
#pragma unroll
            for (int u = 0; u < FIN_BATCH; u++) {
                off[u] = r < rows ? r * pitch + c * V : -1;
                if (r < rows) {
                    const float *p = Gd + (int64_t)(row0 + r) * Np + (col0 + c * V);
                    v[u] = V == 4 ? *reinterpret_cast<const float4 *>(p) : make_float4(p[0], 0.f, 0.f, 0.f);
#pragma unroll
                    for (int s = 1; s < TC_MAX_KSPLIT; s++) {
                        if (s >= planes) break;
                        const float *ps = p + s * plane;
                        const float4 w = V == 4 ? *reinterpret_cast<const float4 *>(ps) : make_float4(ps[0], 0.f, 0.f, 0.f);
                        v[u].x += w.x; v[u].y += w.y; v[u].z += w.z; v[u].w += w.w;
                    }
                }
                c += dc; r += dr;
                if (c >= nv) { c -= nv; r++; }
            }
#pragma unroll
            for (int u = 0; u < FIN_BATCH; u++) {
                if (off[u] < 0) break;
                float *d = dst + off[u];
                d[0] = v[u].x;
                if (V == 4) { d[1] = v[u].y; d[2] = v[u].z; d[3] = v[u].w; }
            }
        }
    };
    stage(sA, i0 * q, wi, j0 * q, wj);
    stage(sB, j0 * q, wj, i0 * q, wi);
    __syncthreads();
    const int qq = q * q;
    const int sj = FIN_THREADS / qq, sa = (FIN_THREADS % qq) / q, sb = FIN_THREADS % q;
    for (int ii = 0; ii * q < wi; ii++) {
        const int i = i0 + ii, jlo = max(j0, i + 1);
        const int n = (j0 + wj / q - jlo) * qq;
        if (n <= 0) continue;
        float *out = gJ + ((int64_t)i * (2 * L - i - 1) / 2 + (jlo - i - 1)) * qq;
        // element e = (jj - jlo + j0) q^2 + a q + b; (jj, a, b) advance by FIN_THREADS = sj q^2 + sa q + sb per step
        int jj = jlo - j0 + threadIdx.x / qq, a = (threadIdx.x % qq) / q, b = threadIdx.x % q;
        for (int e = threadIdx.x; e < n; e += FIN_THREADS) {
            const float v1 = sB[(jj * q + b) * pitch + ii * q + a];
            const float v2 = sA[(ii * q + a) * pitch + jj * q + b];
            out[e] = scale * (v1 + v2);
            b += sb; a += sa; jj += sj;
            if (b >= q) { b -= q; a++; }
            if (a >= q) { a -= q; jj++; }
        }
    }
}

// ---- host side ---------------------------------------------------------------------------------------
// tuning hooks for parameter sweeps (read once; the defaults below are what the product uses)
static int env_int_once(const char *name, int *cache)
{
    if (*cache == -2) {
        const char *e = getenv(name);
        *cache = e ? atoi(e) : -1;
    }
    return *cache;
}

// ring depth for a given stage size: as many stages as fit in the 227 KB opt-in shared memory
static int stages_for(int stage_bytes)
{
    return std::max(2, std::min(TC_MAX_STAGES, (TC_SMEM_LIMIT - TC_SMEM_HEAD) / stage_bytes));
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                    const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_fn()
{
    static PFN_encodeTiled fn = nullptr;
    if (fn) return fn;
    void *p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess || !p)
        return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(p);
    return fn;
}

static int make_map(CUtensorMap *m, void *base, int64_t rows, int64_t kp, int box_rows)
{
    PFN_encodeTiled fn = get_encode_fn();
    if (!fn) { set_error("cuTensorMapEncodeTiled entry point not available"); return 1; }
    cuuint64_t gdim[2] = {(cuuint64_t)kp, (cuuint64_t)rows};
    cuuint64_t gstride[1] = {(cuuint64_t)kp * 2};
    cuuint32_t box[2] = {(cuuint32_t)TC_BK, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, base, gdim, gstride, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed with code " + std::to_string((int)r)); return 1; }
    return 0;
}

// K slices of the backward product.  Each CTA holds an SM alone, so `units` work units run in ceil(units / SMs)
// waves and a part-filled last wave idles the rest of the GPU for a whole CTA duration.  Slicing K multiplies
// the units and divides their duration: take the smallest slice count in 1..4 whose wave efficiency
// units / (SMs * waves) is >= 0.97, else the most efficient one.  Config 2 (726 tiles on 132 SMs, 5.5 waves)
// gets 2 slices = 11 full waves; L = 500 and L = 800 stay at 1.  No slice is left empty.
static int backward_ksplit(int64_t tiles, int num_kb, int sm_count)
{
    static int ks_env = -2;
    const int e = env_int_once("EVC_KSPLIT", &ks_env);
    int ks = 1;
    if (e > 0) {
        ks = std::min(e, TC_MAX_KSPLIT);
    } else {
        double best = 0.0;
        for (int s = 1; s <= 4 && s <= num_kb; s++) {
            const int64_t units = tiles * s;
            const double eff = (double)units / ((double)sm_count * (double)ceil_div(units, sm_count));
            if (eff >= 0.97) { ks = s; break; }
            if (eff > best) { best = eff; ks = s; }
        }
    }
    ks = std::max(1, std::min(ks, num_kb));
    return (int)ceil_div(num_kb, ceil_div(num_kb, ks));    // slices of ceil(num_kb / ks) blocks, none empty
}

int64_t plm_seq_chunk_round(int64_t seq_chunk) { return seq_chunk <= 0 ? 0 : round_up(seq_chunk, PLM_SEQ_CHUNK_ALIGN); }

void plm_tc_geometry(const PlmGeom &g, int sm_count, int64_t seq_chunk, PlmTcGeom &t)
{
    const int64_t lq = (int64_t)g.L * g.q;
    const int64_t c = plm_seq_chunk_round(seq_chunk);
    t.C = (c == 0 || c >= g.N) ? g.N : c;
    t.n_chunks = (int)ceil_div(g.N, t.C);
    t.Mp = round_up(lq, TC_BM);
    t.Np = round_up(lq, TC_BN);
    t.Kp = round_up(t.C, TC_BK);
    const int64_t tiles = (t.Mp / TC_BM) * (t.Np / TC_BN);
    t.ksplit = backward_ksplit(tiles, (int)(t.Kp / TC_BK), sm_count);
    t.ksplit_last = backward_ksplit(tiles, (int)(t.kp_chunk(t.n_chunks - 1, g.N) / TC_BK), sm_count);
    t.planes = std::max(t.ksplit, t.ksplit_last);
}

// Xt for the sequences [n0, n0 + Kp): every column is written (exact zeros beyond N); the rows (j,b) >= L q of the
// M padding are not (zeroed once at allocation)
int plm_tc_build_xt(const PlmGeom &g, const PlmTcGeom &t, const uint32_t *d_msa4, void *d_xt, int64_t n0,
                    cudaStream_t st)
{
    dim3 grid((unsigned)ceil_div(t.Kp, 256), (unsigned)g.L);
    build_xt_kernel<<<grid, 256, 0, st>>>(d_msa4, reinterpret_cast<__nv_bfloat16 *>(d_xt), n0, g.N, g.Nld, t.Kp,
                                          g.L, g.q);
    EVC_KERNEL_CHECK();
    return 0;
}

int plm_tc_make_maps(const PlmTcGeom &t, void *d_xt, void *d_rt_hi, void *d_rt_lo, void *maps_out)
{
    CUtensorMap *m = reinterpret_cast<CUtensorMap *>(maps_out);
    if (make_map(&m[0], d_xt, t.Mp, t.Kp, TC_BM)) return 1;
    if (make_map(&m[1], d_rt_hi, t.Np, t.Kp, TC_BN)) return 1;
    if (make_map(&m[2], d_rt_lo, t.Np, t.Kp, TC_BN)) return 1;
    return 0;
}

// Backward product of sequence chunk `chunk` (0 when the shard is one chunk).  Its K extent is the chunk's real
// sequences rounded up to the K block, so the last, partial chunk reads no stale column beyond that.  Chunk 0 stores
// its planes; a later chunk adds into the planes an earlier chunk wrote (ACC) and stores the others.
int plm_tc_backward(const PlmGeom &g, const PlmTcGeom &t, const void *maps, float *d_Gd, int single, int chunk,
                    cudaStream_t st)
{
    const CUtensorMap *m = reinterpret_cast<const CUtensorMap *>(maps);
    const int stage = TC_A_BYTES + TC_B_BYTES + (single ? 0 : TC_B_BYTES);
    const int n_stages = stages_for(stage);
    const size_t smem = (size_t)n_stages * stage + TC_SMEM_HEAD;
    static int kc_env = -2;
    const int kc = env_int_once("EVC_KCHUNK", &kc_env);
    const int k_chunk = kc > 0 ? kc : TC_K_CHUNK;
    const int m_tiles = (int)(t.Mp / TC_BM), n_tiles = (int)(t.Np / TC_BN);
    const bool last = chunk == t.n_chunks - 1;
    const int ksplit = last ? t.ksplit_last : t.ksplit;
    const int num_kb = (int)(t.kp_chunk(chunk, g.N) / TC_BK);
    const int grid = m_tiles * n_tiles * ksplit;      // ksplit planes of Gd, one per K slice
    const int64_t plane = t.Mp * t.Np;
    if (chunk == 0) {
        if (single) {
            EVC_CUDA(cudaFuncSetAttribute(tc_gemm_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_LIMIT));
            tc_gemm_kernel<1><<<grid, TC_THREADS, smem, st>>>(m[0], m[1], m[2], d_Gd, t.Np, m_tiles, n_tiles,
                                                                num_kb, k_chunk, m_tiles, n_stages, ksplit, plane, 0);
        } else {
            EVC_CUDA(cudaFuncSetAttribute(tc_gemm_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_LIMIT));
            tc_gemm_kernel<0><<<grid, TC_THREADS, smem, st>>>(m[0], m[1], m[2], d_Gd, t.Np, m_tiles, n_tiles,
                                                                num_kb, k_chunk, m_tiles, n_stages, ksplit, plane, 0);
        }
    } else {
        const int acc_planes = t.ksplit;              // chunks 0 .. n_chunks - 2 all wrote t.ksplit planes
        if (single) {
            EVC_CUDA(cudaFuncSetAttribute(tc_gemm_kernel<1, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_LIMIT));
            tc_gemm_kernel<1, 1><<<grid, TC_THREADS, smem, st>>>(m[0], m[1], m[2], d_Gd, t.Np, m_tiles, n_tiles,
                                                                   num_kb, k_chunk, m_tiles, n_stages, ksplit, plane,
                                                                   acc_planes);
        } else {
            EVC_CUDA(cudaFuncSetAttribute(tc_gemm_kernel<0, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_LIMIT));
            tc_gemm_kernel<0, 1><<<grid, TC_THREADS, smem, st>>>(m[0], m[1], m[2], d_Gd, t.Np, m_tiles, n_tiles,
                                                                   num_kb, k_chunk, m_tiles, n_stages, ksplit, plane,
                                                                   acc_planes);
        }
    }
    EVC_KERNEL_CHECK();
    return 0;
}

int plm_tc_finalize_pairs(const PlmGeom &g, const PlmTcGeom &t, const float *d_Gd, int planes, float *d_gJ,
                          float scale, cudaStream_t st)
{
    const unsigned nt = (unsigned)ceil_div(g.L, FIN_SITES);
    auto kernel = g.q > 21 ? finalize_pairs_tc_kernel<true> : finalize_pairs_tc_kernel<false>;
    const int smem = fin_smem_bytes(g.q);
    EVC_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    kernel<<<dim3(nt, nt), FIN_THREADS, smem, st>>>(d_Gd, planes, t.Mp * t.Np, d_gJ, g.L, g.q, (int)t.Np, scale,
                                                    fin_pitch(g.q));
    EVC_KERNEL_CHECK();
    return 0;
}

// ---- tensor-core forward -----------------------------------------------------------------------------
void plm_tcf_geometry(const PlmGeom &g, const PlmTcGeom &tc, PlmTcfGeom &t)
{
    const int64_t lq = (int64_t)g.L * g.q;
    t.Mp = round_up(lq, TC_BM);          // rows of Wt / Zt
    t.Kw = round_up(lq, TC_BK);          // K extent (j,b)
    t.Ns = round_up(tc.C, TC_BN);        // sequences of a chunk rounded to the 192-column tile
    t.Xrows = round_up(tc.C, 384);       // allocation of X: covers 128- and 192-row tilings
    t.ntiles_s = (int)ceil_div(g.N, 256);  // partial-sum tiles of the whole shard
}

// X for the sequences [n0, n0 + Xrows): every row is written (exact zeros beyond N); the K padding is not (zeroed
// once at allocation)
int plm_tcf_build_x(const PlmGeom &g, const PlmTcfGeom &t, const uint32_t *d_msa4, void *d_x1h, int64_t n0,
                    cudaStream_t st)
{
    build_x_kernel<<<(unsigned)t.Xrows, 256, 0, st>>>(d_msa4, reinterpret_cast<__nv_bfloat16 *>(d_x1h), n0,
                                                    std::min(t.Xrows, g.N - n0), g.Nld, g.L, g.q, t.Kw);
    EVC_KERNEL_CHECK();
    return 0;
}

// the two coupling operands of the sparse forward, in boxes of 96 rows (half a state tile: one CTA's share of a
// W stage in a 2-CTA cluster)
int plm_tcf_make_maps(const PlmTcfGeom &t, void *d_wt_hi, void *d_wt_lo, void *maps_out)
{
    CUtensorMap *m = reinterpret_cast<CUtensorMap *>(maps_out);
    if (make_map(&m[0], d_wt_hi, t.Mp, t.Kw, TC_BN / 2)) return 1;
    if (make_map(&m[1], d_wt_lo, t.Mp, t.Kw, TC_BN / 2)) return 1;
    return 0;
}

// the one-hot operand of the sequences [n0, n0 + Xrows) in the fragment-ready 2:4 form (tc_sparse_logits_kernel):
// Xrows / 128 * Kw / 64 * 10240 bytes of the Xrows * Kw * 2 allocated, every byte of them written
int plm_tcf_build_xsp(const PlmGeom &g, const PlmTcfGeom &t, const uint32_t *d_msa4, void *d_x1h, int64_t n0,
                      cudaStream_t st)
{
    const int num_kb = (int)(t.Kw / TC_BK);
    const int64_t n_frag = t.Xrows / TC_BM * num_kb * 4;
    build_xsp_kernel<<<(unsigned)ceil_div(n_frag * 128, 256), 256, 0, st>>>(
        d_msa4, reinterpret_cast<unsigned char *>(d_x1h), n0, std::min(t.Xrows, g.N - n0), g.Nld, g.L, g.q, num_kb,
        n_frag);
    EVC_KERNEL_CHECK();
    return 0;
}

int plm_tcf_expand(const PlmGeom &g, const PlmTcfGeom &t, const float *d_x, void *d_wt_hi, void *d_wt_lo,
                   int single, cudaStream_t st)
{
    const unsigned nt = (unsigned)ceil_div(g.L, EXP_SITES);
    if (g.q > EXP_STATIC_Q) {
        const size_t smem = exp_wide_smem(g.q);
        EVC_CUDA(cudaFuncSetAttribute(expand_tc_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)smem));
        expand_tc_kernel<false, true><<<dim3(nt, nt), EXP_THREADS, smem, st>>>(
            d_x, reinterpret_cast<__nv_bfloat16 *>(d_wt_hi), reinterpret_cast<__nv_bfloat16 *>(d_wt_lo), g.L, g.q,
            t.Kw, single);
        EVC_KERNEL_CHECK();
        return 0;
    }
    expand_tc_kernel<false><<<dim3(nt, nt), EXP_THREADS, 0, st>>>(d_x, reinterpret_cast<__nv_bfloat16 *>(d_wt_hi),
                                                                  reinterpret_cast<__nv_bfloat16 *>(d_wt_lo), g.L, g.q,
                                                                  t.Kw, single);
    EVC_KERNEL_CHECK();
    return 0;
}

// State tiles per group of the forward tile order: the group's slice of the coupling operand (hi [+ lo], all of
// K) should stay L2-resident while every sequence tile passes by.  24 MB per group measured best at config 2
// (71 MB operand, DESIGN.md 4c); long alignments (L = 500: 441 MB) get proportionally fewer tiles per group.
// EVC_MGROUP sets the tile count, EVC_MGROUP_MB the byte budget.
static int forward_group(const PlmTcfGeom &t, int single, int tiles)
{
    static int mg_env = -2;
    const int e = env_int_once("EVC_MGROUP", &mg_env);
    if (e > 0) return std::min(e, tiles);
    static int mb_env = -2;
    const int mb = env_int_once("EVC_MGROUP_MB", &mb_env);
    const double budget = (mb > 0 ? mb : 24) * 1.0e6;
    const double per_tile = (double)TC_BN * (double)t.Kw * 2.0 * (single ? 1.0 : 2.0);
    return std::max(1, std::min(tiles, (int)(budget / per_tile)));
}

// CTAs per cluster of the sparse forward (EVC_FWD_CLUSTER = 1 or 2, read once): 2 halves the L2 -> SM traffic of
// the coupling operand (DESIGN.md 4)
static int forward_cluster()
{
    static int cl_env = -2;
    const int e = env_int_once("EVC_FWD_CLUSTER", &cl_env);
    return e == 1 ? 1 : 2;
}

// Sequences per CTA of the sparse forward: 256 (PAIR) when K is one accumulation chain, else 128.  EVC_FWD_TILE=128
// (read once) forces 128 rows, for comparing the two kernels.
static bool forward_pair(int num_kb, int kchunk)
{
    static int tile_env = -2;
    const int e = env_int_once("EVC_FWD_TILE", &tile_env);
    return e != 128 && kchunk >= num_kb;
}

// logits of `nreal` sequences (the chunk's real ones): only the 128-sequence tiles that hold them are computed
int plm_tcf_logits(const PlmGeom &g, const PlmTcfGeom &t, const void *maps, const void *d_x1h, float *d_zt,
                   int single, int64_t nreal, cudaStream_t st)
{
    const CUtensorMap *m = reinterpret_cast<const CUtensorMap *>(maps);
    const int num_kb = (int)(t.Kw / TC_BK);
    const int kchunk = num_kb <= 128 ? num_kb : TC_K_CHUNK;
    const bool pair = forward_pair(num_kb, kchunk);
    const int stage = TC_B_BYTES + (pair ? 2 : 1) * XSP_KB_BYTES + (single ? 0 : TC_B_BYTES);
    const int n_stages = stages_for(stage);
    const size_t smem = (size_t)n_stages * stage + TC_SMEM_HEAD;
    const int cs = forward_cluster();
    const int state_tiles = (int)ceil_div((int64_t)g.L * g.q, TC_BN);
    const int seq_tiles = (int)ceil_div(nreal, TC_BM);
    const int seq_units = (int)ceil_div(ceil_div(seq_tiles, pair ? 2 : 1), cs);
    const int group = forward_group(t, single, state_tiles);
    auto kernel = pair ? (single ? tc_sparse_logits_kernel<1, 1> : tc_sparse_logits_kernel<0, 1>)
                       : (single ? tc_sparse_logits_kernel<1, 0> : tc_sparse_logits_kernel<0, 0>);
    EVC_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_LIMIT));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(state_tiles * seq_units * cs));
    cfg.blockDim = dim3(TC_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)cs;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    EVC_CUDA(cudaLaunchKernelEx(&cfg, kernel, m[0], m[1], reinterpret_cast<const unsigned char *>(d_x1h), d_zt, t.Ns,
                                t.Mp, state_tiles, seq_tiles, seq_units, num_kb, kchunk, group, n_stages));
    EVC_KERNEL_CHECK();
    return 0;
}

// softmax / residual kernel; d_rt_lo == nullptr in the bf16x1 precision mode (no lo operand is written)
// grid: the 256-sequence tiles of the chunk [n0, n0 + nreal); ntiles = tiles of the whole shard (partial stride)
template <bool ONEHOT>
static int launch_softmax(const PlmGeom &g, int ntiles, const float *d_zt, int64_t ldz, const float *d_x,
                          const uint32_t *d_msa4, const float *d_wts, __nv_bfloat16 *hi, __nv_bfloat16 *lo,
                          int64_t Kp, float *d_gh_part, double *d_fx_part, int64_t n0, int64_t nreal, cudaStream_t st)
{
    dim3 grid((unsigned)ceil_div(nreal, 256), (unsigned)g.L);
    switch (g.q) {
        case 21: plm_softmax_kernel<21, ONEHOT><<<grid, 128, 0, st>>>(d_zt, ldz, d_x, d_msa4, d_wts, hi, lo, Kp, d_gh_part, d_fx_part, g, ntiles, n0); break;
        case 20: plm_softmax_kernel<20, ONEHOT><<<grid, 128, 0, st>>>(d_zt, ldz, d_x, d_msa4, d_wts, hi, lo, Kp, d_gh_part, d_fx_part, g, ntiles, n0); break;
        case 5: plm_softmax_kernel<5, ONEHOT><<<grid, 128, 0, st>>>(d_zt, ldz, d_x, d_msa4, d_wts, hi, lo, Kp, d_gh_part, d_fx_part, g, ntiles, n0); break;
        case 4: plm_softmax_kernel<4, ONEHOT><<<grid, 128, 0, st>>>(d_zt, ldz, d_x, d_msa4, d_wts, hi, lo, Kp, d_gh_part, d_fx_part, g, ntiles, n0); break;
        default:
            // every other alphabet: q states in registers for 8, 16 or 32
            if (g.q < 2 || g.q > PLM_MAX_Q) { set_error("plm softmax kernel: unsupported q"); return 1; }
            if (g.q <= 8)
                plm_softmax_kernel<8, ONEHOT, true><<<grid, 128, 0, st>>>(d_zt, ldz, d_x, d_msa4, d_wts, hi, lo, Kp, d_gh_part, d_fx_part, g, ntiles, n0);
            else if (g.q <= 16)
                plm_softmax_kernel<16, ONEHOT, true><<<grid, 128, 0, st>>>(d_zt, ldz, d_x, d_msa4, d_wts, hi, lo, Kp, d_gh_part, d_fx_part, g, ntiles, n0);
            else
                plm_softmax_kernel<32, ONEHOT, true><<<grid, 128, 0, st>>>(d_zt, ldz, d_x, d_msa4, d_wts, hi, lo, Kp, d_gh_part, d_fx_part, g, ntiles, n0);
    }
    EVC_KERNEL_CHECK();
    return 0;
}

int plm_tcf_softmax(const PlmGeom &g, const PlmTcfGeom &t, const float *d_zt, const float *d_x,
                    const uint32_t *d_msa4, const float *d_wts, void *d_rt_hi, void *d_rt_lo, int64_t Kp,
                    float *d_gh_part, double *d_fx_part, int64_t n0, int64_t nreal, cudaStream_t st)
{
    return launch_softmax<false>(g, t.ntiles_s, d_zt, t.Ns, d_x, d_msa4, d_wts,
                                 reinterpret_cast<__nv_bfloat16 *>(d_rt_hi), reinterpret_cast<__nv_bfloat16 *>(d_rt_lo),
                                 Kp, d_gh_part, d_fx_part, n0, nreal, st);
}

// a6 on the tensor cores: Rt = w_n [s_ni = a] as bf16 hi + lo (the weights keep 16 mantissa bits), per-tile
// partials of f_i; the caller then runs the backward product and symmetrises with scale 0.5
int plm_tc_onehot_residual(const PlmGeom &g, int ntiles, const uint32_t *d_msa4, const float *d_wts, void *d_rt_hi,
                           void *d_rt_lo, int64_t Kp, float *d_gh_part, double *d_fx_part, int64_t n0, int64_t nreal,
                           cudaStream_t st)
{
    return launch_softmax<true>(g, ntiles, nullptr, 0, nullptr, d_msa4, d_wts,
                                reinterpret_cast<__nv_bfloat16 *>(d_rt_hi), reinterpret_cast<__nv_bfloat16 *>(d_rt_lo),
                                Kp, d_gh_part, d_fx_part, n0, nreal, st);
}

// ---- fused tensor-core forward ------------------------------------------------------------------------
void plm_tcff_geometry(const PlmGeom &g, PlmTcffGeom &t)
{
    t.n_tiles = (int)ceil_div(g.L, TF_SITES);
    t.Np = (int64_t)t.n_tiles * TF_BN;
    t.Kw = round_up((int64_t)g.L * g.q, TC_BK);
    t.m_tiles = (int)ceil_div(g.N, TC_BM);
    t.Xrows = round_up(g.N, 384);                  // covers both the 128-row and the 192-row tilings of X
    t.ntile_part = t.m_tiles * 4;
}

bool plm_tcff_supported(const PlmGeom &g) { return g.S == 21; }

int plm_tcff_make_maps(const PlmTcffGeom &t, void *d_x1h, void *d_wp_hi, void *d_wp_lo, void *maps_out)
{
    CUtensorMap *m = reinterpret_cast<CUtensorMap *>(maps_out);
    if (make_map(&m[0], d_x1h, t.Xrows, t.Kw, TC_BM)) return 1;
    if (make_map(&m[1], d_wp_hi, t.Np, t.Kw, TF_BN)) return 1;
    if (make_map(&m[2], d_wp_lo, t.Np, t.Kw, TF_BN)) return 1;
    return 0;
}

int plm_tcff_expand(const PlmGeom &g, const PlmTcffGeom &t, const float *d_x, void *d_wp_hi, void *d_wp_lo,
                    int single, cudaStream_t st)
{
    const unsigned nt = (unsigned)ceil_div(g.L, EXP_SITES);
    expand_tc_kernel<true><<<dim3(nt, nt), EXP_THREADS, 0, st>>>(d_x, reinterpret_cast<__nv_bfloat16 *>(d_wp_hi),
                                                                 reinterpret_cast<__nv_bfloat16 *>(d_wp_lo), g.L, g.q,
                                                                 t.Kw, single);
    EVC_KERNEL_CHECK();
    return 0;
}

int plm_tcff_forward(const PlmGeom &g, const PlmTcffGeom &t, const void *maps, const float *d_x,
                     const uint32_t *d_msa4, const float *d_wts, void *d_rt_hi, void *d_rt_lo, int64_t Kp,
                     float *d_gh_part, double *d_fx_part, int single, cudaStream_t st)
{
    const CUtensorMap *m = reinterpret_cast<const CUtensorMap *>(maps);
    const int stage = TC_A_BYTES + TF_B_BYTES + (single ? 0 : TF_B_BYTES);
    const int n_stages = stages_for(stage);
    const size_t smem = (size_t)n_stages * stage + TC_SMEM_HEAD;
    const int grid = t.m_tiles * t.n_tiles;
    auto kernel = single ? tc_fwd_fused_kernel<1> : tc_fwd_fused_kernel<0>;
    EVC_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_LIMIT));
    kernel<<<grid, TC_THREADS, smem, st>>>(m[0], m[1], m[2], d_x, d_msa4, d_wts, reinterpret_cast<__nv_bfloat16 *>(d_rt_hi),
                                           reinterpret_cast<__nv_bfloat16 *>(d_rt_lo), Kp, d_gh_part, d_fx_part, g,
                                           t.m_tiles, t.n_tiles, (int)(t.Kw / TC_BK), n_stages);
    EVC_KERNEL_CHECK();
    return 0;
}

size_t plm_tc_map_bytes() { return 3 * sizeof(CUtensorMap); }

}  // namespace evc
