// C ABI of libevcplm (declared in include/evcplm.h).  This is the boundary a binding of the
// reference's plmc call site (evcouplings/couplings/tools.py:202-266) talks to.
#include "../../include/evcplm.h"

#include <stdlib.h>

#include <algorithm>
#include <new>
#include <string>
#include <vector>

#include "common.cuh"
#include "internal.h"

namespace evc {
static thread_local std::string g_err;
void set_error(const std::string &msg) { g_err = msg; }
}  // namespace evc

using namespace evc;

static cudaStream_t as_stream(void *s) { return reinterpret_cast<cudaStream_t>(s); }

static const char SUPPORTED_Q[] =
    "supported: 2 <= q <= 32 states with the gap as a state, 2 <= q <= 31 with the ignored gap coded q; "
    "every code must be below 32, the 5 bit-planes of the Hamming pass";

// The gather objective kernels (plm_gather.cu) exist for q in {4, 5, 20, 21} only; every other alphabet runs on the
// tensor-core path.
static int require_gather_q(const evc_plm *h, const char *what)
{
    if (plm_gather_supported_q(h->g.q)) return 0;
    set_error(std::string(what) + ": the gather kernels support q in {4, 5, 20, 21} only, this handle has q=" +
              std::to_string(h->g.q) + "; select the tensor-core path with evc_plm_set_forward(h, 1)");
    return 1;
}

// ---- sizes of the handle's device buffers (shared by the allocations and evc_plm_tc_bytes) ---------------------
static void plm_geom_init(PlmGeom &g, int64_t N, int L, int q, int gap_code)
{
    g.N = N;
    g.L = L;
    g.Lp = (int)round_up(L, 4);
    g.q = q;
    g.gap_code = gap_code;
    g.QB = gap_code >= 0 ? q + 1 : q;
    g.S = (q % 2) ? q : q + 1;
    g.Nr = round_up(N, PLM_BWD_TS);
    g.Nld = round_up(N, 32);
    g.L4 = g.Lp / 4;
    g.ntiles_f = (int)ceil_div(N, PLM_FWD_TS);
    g.ntiles_b = (int)ceil_div(N, PLM_BWD_TS);
    g.n_params = (int64_t)L * q + (int64_t)L * (L - 1) / 2 * q * q;
}
struct HandleBytes {           // evc_plm_create: codes, packed MSA, weights
    size_t codes, msa4, wts;
    explicit HandleBytes(const PlmGeom &g)
        : codes((size_t)g.N * g.L), msa4((size_t)g.L4 * g.Nld * sizeof(uint32_t)), wts((size_t)g.N * sizeof(float)) {}
};
struct TcBwdBytes {            // evc_plm_set_backward(1): Xt, Rt_hi / Rt_lo (each), the Gd planes
    size_t xt, rt, gd;
    explicit TcBwdBytes(const PlmTcGeom &t)
        : xt((size_t)t.Mp * t.Kp * 2), rt((size_t)t.Np * t.Kp * 2), gd((size_t)t.planes * t.Mp * t.Np * sizeof(float)) {}
};
struct TcFwdBytes {            // evc_plm_set_forward(1): X, Wt_hi / Wt_lo (each), Zt, g_h and fx partials
    size_t x, wt, zt, gh_part, fx_part;
    TcFwdBytes(const PlmGeom &g, const PlmTcfGeom &t)
        : x((size_t)t.Xrows * t.Kw * 2), wt((size_t)t.Mp * t.Kw * 2), zt((size_t)t.Mp * t.Ns * sizeof(float)),
          gh_part((size_t)g.L * t.ntiles_s * g.S * sizeof(float)), fx_part((size_t)g.L * t.ntiles_s * sizeof(double)) {}
};

// cudaMalloc that keeps the handle's byte count (evc_plm_device_bytes)
template <class T>
static bool dalloc(evc_plm *h, T **p, size_t bytes)
{
    if (cudaMalloc(p, bytes) != cudaSuccess) return false;
    h->bytes += (int64_t)bytes;
    return true;
}

extern "C" {

int evc_abi_version(void) { return EVCPLM_ABI_VERSION; }

const char *evc_last_error(void) { return g_err.c_str(); }

int evc_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        set_error("cudaGetDeviceCount failed (no CUDA device / driver?)");
        return -1;
    }
    return n;
}

int evc_device_info(int32_t device, int32_t *sm_count, int32_t *cc_major, int32_t *cc_minor,
                    int64_t *total_mem_bytes)
{
    cudaDeviceProp p;
    EVC_CUDA(cudaGetDeviceProperties(&p, device));
    if (sm_count) *sm_count = p.multiProcessorCount;
    if (cc_major) *cc_major = p.major;
    if (cc_minor) *cc_minor = p.minor;
    if (total_mem_bytes) *total_mem_bytes = (int64_t)p.totalGlobalMem;
    return 0;
}

// ---- (b) Hamming ---------------------------------------------------------------------------------
int64_t evc_hamming_plane_words(int64_t N, int32_t L) { return hamming_plane_words(N, L); }
int64_t evc_hamming_num_tiles(int64_t N) { return hamming_num_tiles(N); }

int evc_hamming_pack(const uint8_t *d_codes, int64_t N, int32_t L, uint32_t *d_planes, void *stream)
{
    return hamming_pack(d_codes, N, L, d_planes, as_stream(stream));
}

int evc_hamming_count_tiles(const uint32_t *d_planes, int64_t N, int32_t L, int32_t min_identical,
                            int64_t tile_begin, int64_t tile_end, int32_t *d_counts, void *stream)
{
    return hamming_count_tiles(d_planes, nullptr, N, L, min_identical, tile_begin, tile_end, d_counts,
                               as_stream(stream));
}

int evc_hamming_count_tiles_mult(const uint32_t *d_planes, const int32_t *d_mult, int64_t N, int32_t L,
                                 int32_t min_identical, int64_t tile_begin, int64_t tile_end, int32_t *d_counts,
                                 void *stream)
{
    if (!d_mult) { set_error("evc_hamming_count_tiles_mult: null multiplicities"); return 1; }
    return hamming_count_tiles(d_planes, d_mult, N, L, min_identical, tile_begin, tile_end, d_counts,
                               as_stream(stream));
}

// evc_hamming_counts (mult == nullptr) and evc_hamming_counts_mult; `fn` prefixes the error messages
static int hamming_counts_host(const char *fn, const uint8_t *codes, const int32_t *mult, int64_t N, int32_t L,
                               int32_t min_identical, int32_t device, int32_t *counts_out)
{
    const std::string name(fn);
    if (!codes || !counts_out || N <= 0 || L <= 0) {
        set_error(name + ": empty alignment or null pointer");
        return 1;
    }
    {
        // the pass compares 5 bit-planes: a code >= 32 would alias a smaller one
        unsigned mx = 0;
        const size_t total = (size_t)N * L;
        for (size_t e = 0; e < total; e++) mx = codes[e] > mx ? codes[e] : mx;
        if (mx >= 32) {
            set_error(name + ": sequence code " + std::to_string(mx) + " out of range (codes must be < 32)");
            return 1;
        }
    }
    if (mult) {
        // a count is at most the sum of the multiplicities, and the counters are int32
        int64_t sum = 0;
        for (int64_t r = 0; r < N; r++) {
            if (mult[r] < 1) { set_error(name + ": multiplicities must be >= 1"); return 1; }
            sum += mult[r];
        }
        if (sum > INT32_MAX) { set_error(name + ": the multiplicities sum to more than 2^31 - 1"); return 1; }
    }
    EVC_CUDA(cudaSetDevice(device));
    uint8_t *d_codes = nullptr;
    uint32_t *d_planes = nullptr;
    int32_t *d_counts = nullptr, *d_mult = nullptr;
    int rc = 1;
    do {
        if (cudaMalloc(&d_codes, (size_t)N * L) != cudaSuccess ||
            cudaMalloc(&d_planes, (size_t)hamming_plane_words(N, L) * sizeof(uint32_t)) != cudaSuccess ||
            cudaMalloc(&d_counts, (size_t)N * sizeof(int32_t)) != cudaSuccess ||
            (mult && cudaMalloc(&d_mult, (size_t)N * sizeof(int32_t)) != cudaSuccess)) {
            set_error(name + ": device allocation failed");
            break;
        }
        if (cudaMemcpy(d_codes, codes, (size_t)N * L, cudaMemcpyHostToDevice) != cudaSuccess ||
            (mult && cudaMemcpy(d_mult, mult, (size_t)N * sizeof(int32_t), cudaMemcpyHostToDevice) != cudaSuccess) ||
            cudaMemset(d_counts, 0, (size_t)N * sizeof(int32_t)) != cudaSuccess) {
            set_error(name + ": H2D failed");
            break;
        }
        if (hamming_pack(d_codes, N, L, d_planes, 0)) break;
        if (hamming_count_tiles(d_planes, d_mult, N, L, min_identical, 0, hamming_num_tiles(N), d_counts, 0)) break;
        if (cudaMemcpy(counts_out, d_counts, (size_t)N * sizeof(int32_t), cudaMemcpyDeviceToHost) !=
            cudaSuccess) {
            set_error(name + ": kernel/D2H failed: " + cudaGetErrorString(cudaGetLastError()));
            break;
        }
        rc = 0;
    } while (0);
    cudaFree(d_codes);
    cudaFree(d_planes);
    cudaFree(d_counts);
    cudaFree(d_mult);
    return rc;
}

int evc_hamming_counts(const uint8_t *codes, int64_t N, int32_t L, int32_t min_identical, int32_t device,
                       int32_t *counts_out)
{
    return hamming_counts_host("evc_hamming_counts", codes, nullptr, N, L, min_identical, device, counts_out);
}

int evc_hamming_counts_mult(const uint8_t *codes, const int32_t *mult, int64_t N, int32_t L, int32_t min_identical,
                            int32_t device, int32_t *counts_out)
{
    if (!mult) { set_error("evc_hamming_counts_mult: null multiplicities"); return 1; }
    return hamming_counts_host("evc_hamming_counts_mult", codes, mult, N, L, min_identical, device, counts_out);
}

// ---- distinct rows ---------------------------------------------------------------------------------------
int evc_msa_unique(const uint8_t *d_codes, int64_t N, int32_t L, int32_t *d_first, int32_t *d_inverse,
                   int32_t *d_mult, int64_t *U_out, void *stream)
{
    if (!d_codes || !d_first || !d_inverse || !d_mult || !U_out) {
        set_error("evc_msa_unique: null pointer");
        return 1;
    }
    return msa_unique(d_codes, N, L, d_first, d_inverse, d_mult, U_out, as_stream(stream));
}

int evc_msa_unique_host(const uint8_t *codes, int64_t N, int32_t L, int32_t device, int32_t *first_out,
                        int32_t *inverse_out, int32_t *mult_out, int64_t *U_out)
{
    if (!codes || !first_out || !inverse_out || !mult_out || !U_out || N <= 0 || L <= 0) {
        set_error("evc_msa_unique_host: empty alignment or null pointer");
        return 1;
    }
    EVC_CUDA(cudaSetDevice(device));
    uint8_t *d_codes = nullptr;
    int32_t *d_idx = nullptr;
    int rc = 1;
    do {
        if (cudaMalloc(&d_codes, (size_t)N * L) != cudaSuccess ||
            cudaMalloc(&d_idx, (size_t)3 * N * sizeof(int32_t)) != cudaSuccess) {
            set_error("evc_msa_unique_host: device allocation failed");
            break;
        }
        if (cudaMemcpy(d_codes, codes, (size_t)N * L, cudaMemcpyHostToDevice) != cudaSuccess) {
            set_error("evc_msa_unique_host: H2D failed");
            break;
        }
        int64_t U = 0;
        if (msa_unique(d_codes, N, L, d_idx, d_idx + N, d_idx + 2 * N, &U, 0)) break;
        if (cudaMemcpy(first_out, d_idx, (size_t)U * sizeof(int32_t), cudaMemcpyDeviceToHost) != cudaSuccess ||
            cudaMemcpy(inverse_out, d_idx + N, (size_t)N * sizeof(int32_t), cudaMemcpyDeviceToHost) != cudaSuccess ||
            cudaMemcpy(mult_out, d_idx + 2 * N, (size_t)U * sizeof(int32_t), cudaMemcpyDeviceToHost) != cudaSuccess) {
            set_error(std::string("evc_msa_unique_host: D2H failed: ") + cudaGetErrorString(cudaGetLastError()));
            break;
        }
        *U_out = U;
        rc = 0;
    } while (0);
    cudaFree(d_codes);
    cudaFree(d_idx);
    return rc;
}

int evc_identities_to_seq(const uint8_t *d_codes, const uint8_t *d_seq, int64_t N, int32_t L, int32_t *d_out,
                          void *stream)
{
    if (!d_codes || !d_seq || !d_out) { set_error("evc_identities_to_seq: null pointer"); return 1; }
    return identities_to_seq(d_codes, d_seq, N, L, d_out, as_stream(stream));
}

// ---- (a) PLM ---------------------------------------------------------------------------------------
void evc_plm_destroy(evc_plm_t *h)
{
    if (!h) return;
    cudaSetDevice(h->device);
    cudaFree(h->d_codes);
    cudaFree(h->d_msa4);
    cudaFree(h->d_perm);
    cudaFree(h->d_bstart);
    cudaFree(h->d_wts);
    cudaFree(h->d_W);
    cudaFree(h->d_G);
    cudaFree(h->d_R);
    cudaFree(h->d_gh_part);
    cudaFree(h->d_fx_part);
    cudaFree(h->d_x_tmp);
    cudaFree(h->d_g_tmp);
    cudaFree(h->d_fx_tmp);
    cudaFree(h->d_xt);
    cudaFree(h->d_rt_hi);
    cudaFree(h->d_rt_lo);
    cudaFree(h->d_Gd);
    free(h->tc_maps);
    cudaFree(h->d_x1h);
    cudaFree(h->d_wt_hi);
    cudaFree(h->d_wt_lo);
    cudaFree(h->d_zt);
    cudaFree(h->d_gh_part2);
    cudaFree(h->d_fx_part2);
    free(h->tcf_maps);
    cudaFree(h->d_wp_hi);
    cudaFree(h->d_wp_lo);
    cudaFree(h->d_gh_part3);
    cudaFree(h->d_fx_part3);
    free(h->tcff_maps);
    for (int k = 0; k < 6; k++)
        if (h->ev[k]) cudaEventDestroy(h->ev[k]);
    fit_work_free(h->fit);
    delete h;
}

// evc_plm_create (any_q = false: the alphabets q in {4, 5, 20, 21} it has always taken) and
// evc_plm_create_alphabet (any_q = true: every q of plm_supported_q); `fn` prefixes the error messages
static int plm_create(const char *fn, bool any_q, evc_plm_t **out, const uint8_t *codes, int64_t N, int32_t L,
                      int32_t q, int32_t gap_code, const float *weights, int32_t device)
{
    const std::string name(fn);
    if (!out || !codes || !weights) { set_error(name + ": null pointer"); return 1; }
    *out = nullptr;
    if (N <= 0 || L < 2) { set_error(name + ": need N >= 1 sequences and L >= 2 sites"); return 1; }
    if (!any_q && !plm_gather_supported_q(q)) {
        set_error(name + ": unsupported number of states q=" + std::to_string(q) +
                  " (supported: 4, 5, 20, 21; evc_plm_create_alphabet takes 2 <= q <= 32)");
        return 1;
    }
    if (gap_code >= 0 && gap_code != q) {
        set_error(name + ": gap_code must be -1 or q");
        return 1;
    }
    if (!plm_supported_q(q, gap_code)) {
        set_error(name + ": unsupported number of states q=" + std::to_string(q) +
                  (gap_code >= 0 ? " with the ignored gap" : "") + " (" + SUPPORTED_Q + ")");
        return 1;
    }
    if (L > 65535) { set_error(name + ": L too large"); return 1; }
    // every code must address a row of a coupling block: 0..q-1, or q for the ignored gap (the kernels index
    // shared-memory rows with the raw byte, so an out-of-range code would silently read another site's block)
    {
        unsigned mx = 0;
        const size_t total = (size_t)N * L;
        for (size_t e = 0; e < total; e++) mx = codes[e] > mx ? codes[e] : mx;
        if ((int)mx >= (gap_code >= 0 ? q + 1 : q)) {
            set_error(name + ": sequence code " + std::to_string(mx) + " out of range (valid: 0.." +
                      std::to_string((gap_code >= 0 ? q + 1 : q) - 1) + (gap_code >= 0 ? ", the last one being the ignored gap)" : ")"));
            return 1;
        }
    }
    EVC_CUDA(cudaSetDevice(device));
    evc_plm *h = new (std::nothrow) evc_plm();
    if (!h) { set_error(name + ": out of host memory"); return 1; }
    h->device = device;
    PlmGeom &g = h->g;
    plm_geom_init(g, N, L, q, gap_code);
    const HandleBytes hb(g);

    bool ok = dalloc(h, &h->d_codes, hb.codes) && dalloc(h, &h->d_msa4, hb.msa4) && dalloc(h, &h->d_wts, hb.wts);
    if (!ok) {
        set_error(name + ": device allocation failed: " +
                  cudaGetErrorString(cudaGetLastError()));
        evc_plm_destroy(h);
        return 1;
    }
    ok = cudaMemcpy(h->d_codes, codes, (size_t)N * L, cudaMemcpyHostToDevice) == cudaSuccess &&
         cudaMemcpy(h->d_wts, weights, (size_t)N * sizeof(float), cudaMemcpyHostToDevice) == cudaSuccess;
    if (!ok || plm_pack_msa(g, h->d_codes, h->d_msa4, 0) || cudaDeviceSynchronize() != cudaSuccess) {
        if (ok) set_error(name + ": packing failed: " + cudaGetErrorString(cudaGetLastError()));
        else set_error(name + ": H2D failed");
        evc_plm_destroy(h);
        return 1;
    }
    *out = h;
    return 0;
}

int evc_plm_create(evc_plm_t **out, const uint8_t *codes, int64_t N, int32_t L, int32_t q, int32_t gap_code,
                   const float *weights, int32_t device)
{
    return plm_create("evc_plm_create", false, out, codes, N, L, q, gap_code, weights, device);
}

int evc_plm_create_alphabet(evc_plm_t **out, const uint8_t *codes, int64_t N, int32_t L, int32_t q, int32_t gap_code,
                            const float *weights, int32_t device)
{
    return plm_create("evc_plm_create_alphabet", true, out, codes, N, L, q, gap_code, weights, device);
}

// Expanded couplings W and residual buffer R: all the energies need (W, and R as the per-site partials), for any q.
static int ensure_expanded(evc_plm *h)
{
    if (h->expanded_ready) return 0;
    EVC_CUDA(cudaSetDevice(h->device));
    const PlmGeom &g = h->g;
    const size_t w_bytes = (size_t)g.w_floats() * sizeof(float);
    const size_t r_bytes = (size_t)g.L * g.Nr * g.S * sizeof(float);
    if (!dalloc(h, &h->d_W, w_bytes) || !dalloc(h, &h->d_R, r_bytes)) {
        set_error(std::string("libevcplm: device allocation of the expanded couplings failed: ") +
                  cudaGetErrorString(cudaGetLastError()));
        return 1;
    }
    EVC_CUDA(cudaMemset(h->d_W, 0, w_bytes));
    EVC_CUDA(cudaMemset(h->d_R, 0, r_bytes));
    h->expanded_ready = true;
    return 0;
}

// Buffers of the gather path (expanded couplings W, their gradient G, residuals R, state-sorted bucket lists):
// 6.7 GB of R alone at N = 100k, L = 800 -- allocated only when a gather kernel is actually selected.  The bucket
// lists hold at most PLM_BWD_BS - 2 buckets: only the gather alphabets may build them.
static int ensure_gather(evc_plm *h)
{
    if (h->gather_ready) return 0;
    if (require_gather_q(h, "libevcplm")) return 1;
    if (ensure_expanded(h)) return 1;
    const PlmGeom &g = h->g;
    const size_t w_bytes = (size_t)g.w_floats() * sizeof(float);
    const bool ok = dalloc(h, &h->d_perm, (size_t)g.ntiles_b * g.L * PLM_BWD_CAP * sizeof(uint32_t)) &&
                    dalloc(h, &h->d_bstart, (size_t)g.ntiles_b * g.L * PLM_BWD_BS * sizeof(uint16_t)) &&
                    dalloc(h, &h->d_G, w_bytes) &&
                    dalloc(h, &h->d_gh_part, (size_t)g.L * g.ntiles_f * g.S * sizeof(float)) &&
                    dalloc(h, &h->d_fx_part, (size_t)g.L * g.ntiles_f * sizeof(double));
    if (!ok) {
        set_error(std::string("libevcplm: device allocation of the gather-path buffers failed: ") +
                  cudaGetErrorString(cudaGetLastError()));
        return 1;
    }
    if (plm_build_buckets(g, h->d_codes, h->d_perm, h->d_bstart, 0)) return 1;
    EVC_CUDA(cudaDeviceSynchronize());
    h->gather_ready = true;
    return 0;
}

int64_t evc_plm_num_params(const evc_plm_t *h) { return h ? h->g.n_params : -1; }

int evc_plm_set_precision(evc_plm_t *h, int32_t mode)
{
    if (!h) { set_error("evc_plm_set_precision: null handle"); return 1; }
    if (mode != 0 && mode != 1) {
        set_error("evc_plm_set_precision: mode must be 0 (fp32-equivalent, bf16 hi+lo products) or 1 (bf16 tiles)");
        return 1;
    }
    h->precision = mode;
    return 0;
}

int evc_plm_eval_data(evc_plm_t *h, const float *d_x, float *d_g, double *d_fx, void *stream)
{
    if (!h || !d_x || !d_g || !d_fx) { set_error("evc_plm_eval_data: null pointer"); return 1; }
    cudaStream_t st = as_stream(stream);
    const PlmGeom &g = h->g;
    const bool prof = h->profiling;
    const bool tc = h->bwd_mode == 1;
    const bool tcf = h->fwd_mode == 1;
    const bool tcff = h->fwd_mode == 2;
    const int single = h->precision == 1 ? 1 : 0;      // only the tensor-core products have a reduced mode
    void *rt_lo = single ? nullptr : h->d_rt_lo;
    float *gJ = d_g + (int64_t)g.L * g.q;
    if (tc && h->tc.n_chunks > 1) {
        // sequence chunks (evc_plm_set_seq_chunk): expand once; per chunk the one-hot operands of its sequences,
        // the logits GEMM, the softmax and the backward GEMM adding into the Gd planes; the finalizes once.  The
        // per-stage events are not recorded (evc_plm_last_stage_ms reports an error).
        if (!tcf) {
            set_error("evc_plm_eval_data: sequence chunks need the tensor-core forward (evc_plm_set_forward 1)");
            return 1;
        }
        h->ev_valid = false;
        if (plm_tcf_expand(g, h->tcf, d_x, h->d_wt_hi, h->d_wt_lo, single, st)) return 1;
        for (int c = 0; c < h->tc.n_chunks; c++) {
            const int64_t n0 = (int64_t)c * h->tc.C, nreal = std::min(h->tc.C, g.N - n0);
            if (plm_tcf_build_xsp(g, h->tcf, h->d_msa4, h->d_x1h, n0, st)) return 1;
            if (plm_tc_build_xt(g, h->tc, h->d_msa4, h->d_xt, n0, st)) return 1;
            if (plm_tcf_logits(g, h->tcf, h->tcf_maps, h->d_x1h, h->d_zt, single, nreal, st)) return 1;
            if (plm_tcf_softmax(g, h->tcf, h->d_zt, d_x, h->d_msa4, h->d_wts, h->d_rt_hi, rt_lo, h->tc.Kp,
                                h->d_gh_part2, h->d_fx_part2, n0, nreal, st))
                return 1;
            if (plm_tc_backward(g, h->tc, h->tc_maps, h->d_Gd, single, c, st)) return 1;
        }
        if (plm_tc_finalize_pairs(g, h->tc, h->d_Gd, h->tc.planes, gJ, 1.0f, st)) return 1;
        return plm_finalize_fields_n(g, h->d_gh_part2, h->d_fx_part2, d_g, d_fx, h->tcf.ntiles_s, st);
    }
    if (!tc || (!tcf && !tcff)) {
        if (require_gather_q(h, "evc_plm_eval_data") || ensure_gather(h)) return 1;
    }
    if (prof) EVC_CUDA(cudaEventRecord(h->ev[0], st));
    if (tcff) {
        // expand -> fused wgmma forward (logits + softmax + residuals) -> wgmma backward GEMM
        if (plm_tcff_expand(g, h->tcff, d_x, h->d_wp_hi, h->d_wp_lo, single, st)) return 1;
        if (prof) EVC_CUDA(cudaEventRecord(h->ev[1], st));
        if (plm_tcff_forward(g, h->tcff, h->tcff_maps, d_x, h->d_msa4, h->d_wts, h->d_rt_hi, h->d_rt_lo, h->tc.Kp,
                             h->d_gh_part3, h->d_fx_part3, single, st))
            return 1;
        if (prof) {
            EVC_CUDA(cudaEventRecord(h->ev[2], st));
            EVC_CUDA(cudaEventRecord(h->ev[3], st));
        }
        if (plm_tc_backward(g, h->tc, h->tc_maps, h->d_Gd, single, 0, st)) return 1;
        if (prof) EVC_CUDA(cudaEventRecord(h->ev[4], st));
        if (plm_tc_finalize_pairs(g, h->tc, h->d_Gd, h->tc.planes, gJ, 1.0f, st)) return 1;
        if (plm_finalize_fields_n(g, h->d_gh_part3, h->d_fx_part3, d_g, d_fx, h->tcff.ntile_part, st)) return 1;
    } else if (tcf) {
        // expand -> wgmma logits GEMM -> softmax/residuals -> wgmma backward GEMM
        if (plm_tcf_expand(g, h->tcf, d_x, h->d_wt_hi, h->d_wt_lo, single, st)) return 1;
        if (prof) EVC_CUDA(cudaEventRecord(h->ev[1], st));
        if (plm_tcf_logits(g, h->tcf, h->tcf_maps, h->d_x1h, h->d_zt, single, g.N, st)) return 1;
        if (prof) EVC_CUDA(cudaEventRecord(h->ev[2], st));
        if (plm_tcf_softmax(g, h->tcf, h->d_zt, d_x, h->d_msa4, h->d_wts, h->d_rt_hi, rt_lo, h->tc.Kp,
                            h->d_gh_part2, h->d_fx_part2, 0, g.N, st))
            return 1;
        if (prof) EVC_CUDA(cudaEventRecord(h->ev[3], st));
        if (plm_tc_backward(g, h->tc, h->tc_maps, h->d_Gd, single, 0, st)) return 1;
        if (prof) EVC_CUDA(cudaEventRecord(h->ev[4], st));
        if (plm_tc_finalize_pairs(g, h->tc, h->d_Gd, h->tc.planes, gJ, 1.0f, st)) return 1;
        if (plm_finalize_fields_n(g, h->d_gh_part2, h->d_fx_part2, d_g, d_fx, h->tcf.ntiles_s, st)) return 1;
    } else {
        if (plm_expand(g, d_x, h->d_W, st)) return 1;
        if (!tc) EVC_CUDA(cudaMemsetAsync(h->d_G, 0, (size_t)g.w_floats() * sizeof(float), st));
        if (prof) EVC_CUDA(cudaEventRecord(h->ev[1], st));
        if (plm_forward(g, h->d_W, d_x, h->d_msa4, h->d_wts, h->d_R, tc ? h->d_rt_hi : nullptr,
                        tc ? h->d_rt_lo : nullptr, h->tc.Kp, h->d_gh_part, h->d_fx_part, st))
            return 1;
        if (prof) {
            EVC_CUDA(cudaEventRecord(h->ev[2], st));
            EVC_CUDA(cudaEventRecord(h->ev[3], st));
        }
        if (tc) {
            if (plm_tc_backward(g, h->tc, h->tc_maps, h->d_Gd, single, 0, st)) return 1;
            if (prof) EVC_CUDA(cudaEventRecord(h->ev[4], st));
            if (plm_tc_finalize_pairs(g, h->tc, h->d_Gd, h->tc.planes, gJ, 1.0f, st)) return 1;
            if (plm_finalize_fields(g, h->d_gh_part, h->d_fx_part, d_g, d_fx, st)) return 1;
        } else {
            if (plm_backward(g, h->d_R, h->d_perm, h->d_bstart, h->d_G, st)) return 1;
            if (prof) EVC_CUDA(cudaEventRecord(h->ev[4], st));
            if (plm_finalize(g, h->d_G, h->d_gh_part, h->d_fx_part, d_g, gJ, d_fx, 1.0f, st)) return 1;
        }
    }
    if (prof) {
        EVC_CUDA(cudaEventRecord(h->ev[5], st));
        h->ev_valid = true;
    }
    return 0;
}

int evc_plm_set_backward(evc_plm_t *h, int32_t mode)
{
    if (!h) { set_error("evc_plm_set_backward: null handle"); return 1; }
    if (mode != 0 && mode != 1) { set_error("evc_plm_set_backward: mode must be 0 (gather) or 1 (tensor core)"); return 1; }
    if (mode == 0 && require_gather_q(h, "evc_plm_set_backward")) return 1;
    EVC_CUDA(cudaSetDevice(h->device));
    if (mode == 1 && !h->d_xt) {
        int sm_count = 0;
        EVC_CUDA(cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, h->device));
        plm_tc_geometry(h->g, sm_count, h->seq_chunk, h->tc);
        const PlmTcGeom &t = h->tc;
        const TcBwdBytes b(t);
        if (!dalloc(h, &h->d_xt, b.xt) || !dalloc(h, &h->d_rt_hi, b.rt) || !dalloc(h, &h->d_rt_lo, b.rt) ||
            !dalloc(h, &h->d_Gd, b.gd)) {
            set_error(std::string("evc_plm_set_backward: device allocation failed: ") +
                      cudaGetErrorString(cudaGetLastError()));
            return 1;
        }
        EVC_CUDA(cudaMemset(h->d_xt, 0, b.xt));
        EVC_CUDA(cudaMemset(h->d_rt_hi, 0, b.rt));
        EVC_CUDA(cudaMemset(h->d_rt_lo, 0, b.rt));
        EVC_CUDA(cudaMemset(h->d_Gd, 0, b.gd));
        // one chunk: Xt is static; several: it is rebuilt for every chunk of an evaluation
        if (t.n_chunks == 1 && plm_tc_build_xt(h->g, t, h->d_msa4, h->d_xt, 0, 0)) return 1;
        EVC_CUDA(cudaDeviceSynchronize());
        h->tc_maps = aligned_alloc(64, round_up((int64_t)plm_tc_map_bytes(), 64));
        if (!h->tc_maps) { set_error("evc_plm_set_backward: out of host memory"); return 1; }
        if (plm_tc_make_maps(t, h->d_xt, h->d_rt_hi, h->d_rt_lo, h->tc_maps)) return 1;
    }
    h->bwd_mode = mode;
    return 0;
}

int evc_plm_set_forward(evc_plm_t *h, int32_t mode)
{
    if (!h) { set_error("evc_plm_set_forward: null handle"); return 1; }
    if (mode < 0 || mode > 2) {
        set_error("evc_plm_set_forward: mode must be 0 (gather), 1 (tensor core) or 2 (tensor core, fused softmax)");
        return 1;
    }
    if (mode == 0 && require_gather_q(h, "evc_plm_set_forward")) return 1;
    EVC_CUDA(cudaSetDevice(h->device));
    // the fused variant needs the 21-wide site layout and keeps the whole K extent in one register accumulation
    // chain (no K-chunk promotion): nucleotide alphabets and L*q > 8192 use the unfused tensor-core forward
    // ... and it is not chunked: with sequence chunks the fused mode falls back to mode 1 as well
    const int64_t chunk = plm_seq_chunk_round(h->seq_chunk);
    const bool chunked = chunk > 0 && chunk < h->g.N;
    if (mode == 2 && (!plm_tcff_supported(h->g) || (int64_t)h->g.L * h->g.q > 8192 || chunked)) mode = 1;
    if (mode >= 1) {
        if (evc_plm_set_backward(h, 1)) return 1;     // the tensor-core forward feeds the tensor-core backward
        if (!h->d_x1h) {
            plm_tcf_geometry(h->g, h->tc, h->tcf);
            const PlmTcfGeom &t = h->tcf;
            const TcFwdBytes b(h->g, t);
            if (!dalloc(h, &h->d_x1h, b.x)) {
                set_error("evc_plm_set_forward: device allocation failed (one-hot operand)");
                return 1;
            }
            EVC_CUDA(cudaMemset(h->d_x1h, 0, b.x));
        }
        // one chunk: X is static, in the form the selected forward reads (2:4-sparse fragments for mode 1, dense
        // rows for the fused mode 2), rebuilt when the mode switches between them; several chunks (mode 1 only):
        // it is rebuilt for every chunk of an evaluation
        if (h->tc.n_chunks == 1 && h->x1h_form != mode) {
            if (mode == 1 ? plm_tcf_build_xsp(h->g, h->tcf, h->d_msa4, h->d_x1h, 0, 0)
                          : plm_tcf_build_x(h->g, h->tcf, h->d_msa4, h->d_x1h, 0, 0))
                return 1;
            EVC_CUDA(cudaDeviceSynchronize());
            h->x1h_form = mode;
        }
    }
    if (mode == 1 && !h->d_zt) {
        const PlmTcfGeom &t = h->tcf;
        const TcFwdBytes b(h->g, t);
        if (!dalloc(h, &h->d_wt_hi, b.wt) || !dalloc(h, &h->d_wt_lo, b.wt) || !dalloc(h, &h->d_zt, b.zt) ||
            !dalloc(h, &h->d_gh_part2, b.gh_part) || !dalloc(h, &h->d_fx_part2, b.fx_part)) {
            set_error(std::string("evc_plm_set_forward: device allocation failed: ") +
                      cudaGetErrorString(cudaGetLastError()));
            return 1;
        }
        EVC_CUDA(cudaMemset(h->d_wt_hi, 0, b.wt));
        EVC_CUDA(cudaMemset(h->d_wt_lo, 0, b.wt));
        h->tcf_maps = aligned_alloc(64, round_up((int64_t)plm_tc_map_bytes(), 64));
        if (!h->tcf_maps) { set_error("evc_plm_set_forward: out of host memory"); return 1; }
        if (plm_tcf_make_maps(t, h->d_wt_hi, h->d_wt_lo, h->tcf_maps)) return 1;
    }
    if (mode == 2 && !h->d_wp_hi) {
        plm_tcff_geometry(h->g, h->tcff);
        const PlmTcffGeom &t = h->tcff;
        const size_t wb = (size_t)t.Np * t.Kw * 2;
        if (!dalloc(h, &h->d_wp_hi, wb) || !dalloc(h, &h->d_wp_lo, wb) ||
            !dalloc(h, &h->d_gh_part3, (size_t)h->g.L * t.ntile_part * h->g.S * sizeof(float)) ||
            !dalloc(h, &h->d_fx_part3, (size_t)h->g.L * t.ntile_part * sizeof(double))) {
            set_error(std::string("evc_plm_set_forward: device allocation failed: ") +
                      cudaGetErrorString(cudaGetLastError()));
            return 1;
        }
        EVC_CUDA(cudaMemset(h->d_wp_hi, 0, wb));
        EVC_CUDA(cudaMemset(h->d_wp_lo, 0, wb));
        h->tcff_maps = aligned_alloc(64, round_up((int64_t)plm_tc_map_bytes(), 64));
        if (!h->tcff_maps) { set_error("evc_plm_set_forward: out of host memory"); return 1; }
        if (plm_tcff_make_maps(t, h->d_x1h, h->d_wp_hi, h->d_wp_lo, h->tcff_maps)) return 1;
    }
    h->fwd_mode = mode;
    return 0;
}

int evc_plm_set_seq_chunk(evc_plm_t *h, int64_t seq_chunk)
{
    if (!h) { set_error("evc_plm_set_seq_chunk: null handle"); return 1; }
    if (seq_chunk < 0) { set_error("evc_plm_set_seq_chunk: seq_chunk must be >= 0 (0: whole shard)"); return 1; }
    const int64_t c = plm_seq_chunk_round(seq_chunk);
    if (h->d_xt) {
        // the tensor-core buffers are sized for the chunk they were allocated with
        const int64_t have = h->tc.n_chunks > 1 ? h->tc.C : 0;
        const int64_t want = (c > 0 && c < h->g.N) ? c : 0;
        if (have != want) {
            set_error("evc_plm_set_seq_chunk: the tensor-core buffers already exist for " +
                      (have ? std::to_string(have) + " sequences per chunk" : std::string("the whole shard")) +
                      "; set the chunk before evc_plm_set_backward / evc_plm_set_forward");
            return 1;
        }
    }
    h->seq_chunk = c;
    return 0;
}

// evc_plm_tc_bytes (any_q = false: q in {4, 5, 20, 21}, the alphabets of evc_plm_create) and
// evc_plm_tc_bytes_alphabet (any_q = true: the alphabets of evc_plm_create_alphabet)
static int plm_tc_bytes(const char *fn, bool any_q, int64_t N, int32_t L, int32_t q, int32_t gap_code,
                        int64_t seq_chunk, int32_t sm_count, int64_t *bytes_out)
{
    const std::string name(fn);
    if (!bytes_out) { set_error(name + ": null pointer"); return 1; }
    const bool q_ok = any_q ? plm_supported_q(q, gap_code) : plm_gather_supported_q(q);
    if (N <= 0 || L < 2 || L > 65535 || !q_ok || (gap_code >= 0 && gap_code != q) || seq_chunk < 0 ||
        sm_count <= 0) {
        set_error(name + ": invalid arguments (need N >= 1, 2 <= L <= 65535, gap_code -1 or q, seq_chunk >= 0, "
                  "sm_count >= 1; q: " + (any_q ? std::string(SUPPORTED_Q)
                                                : std::string("4, 5, 20 or 21; evc_plm_tc_bytes_alphabet takes "
                                                              "2 <= q <= 32")) + ")");
        return 1;
    }
    PlmGeom g{};
    plm_geom_init(g, N, L, q, gap_code);
    PlmTcGeom t{};
    plm_tc_geometry(g, sm_count, seq_chunk, t);
    PlmTcfGeom f{};
    plm_tcf_geometry(g, t, f);
    const HandleBytes hb(g);
    const TcBwdBytes bb(t);
    const TcFwdBytes fb(g, f);
    *bytes_out = (int64_t)(hb.codes + hb.msa4 + hb.wts + bb.xt + 2 * bb.rt + bb.gd + fb.x + 2 * fb.wt + fb.zt +
                           fb.gh_part + fb.fx_part);
    return 0;
}

int evc_plm_tc_bytes(int64_t N, int32_t L, int32_t q, int32_t gap_code, int64_t seq_chunk, int32_t sm_count,
                     int64_t *bytes_out)
{
    return plm_tc_bytes("evc_plm_tc_bytes", false, N, L, q, gap_code, seq_chunk, sm_count, bytes_out);
}

int evc_plm_tc_bytes_alphabet(int64_t N, int32_t L, int32_t q, int32_t gap_code, int64_t seq_chunk,
                              int32_t sm_count, int64_t *bytes_out)
{
    return plm_tc_bytes("evc_plm_tc_bytes_alphabet", true, N, L, q, gap_code, seq_chunk, sm_count, bytes_out);
}

int64_t evc_plm_device_bytes(const evc_plm_t *h) { return h ? h->bytes + fit_work_bytes(h->fit) : -1; }

// evc_plm_copy_onehot and evc_plm_copy_stage; `fn` prefixes the error messages
static int copy_stage(const char *fn, const evc_plm_t *h, int32_t which, void *dst, int64_t bytes)
{
    const std::string name(fn);
    if (!h || !dst) { set_error(name + ": null pointer"); return 1; }
    const void *src = nullptr;
    int64_t have = 0;
    const char *what = "";
    const bool fused = h->fwd_mode == 2;
    const PlmTcGeom &t = h->tc;
    const PlmTcfGeom &f = h->tcf;
    const PlmTcffGeom &ff = h->tcff;
    switch (which) {
        case EVC_STAGE_WT_HI: src = h->d_wt_hi; have = f.Mp * f.Kw * 2; what = "Wt_hi"; break;
        case EVC_STAGE_WT_LO: src = h->d_wt_lo; have = f.Mp * f.Kw * 2; what = "Wt_lo"; break;
        case EVC_STAGE_WP_HI: src = h->d_wp_hi; have = ff.Np * ff.Kw * 2; what = "Wp_hi"; break;
        case EVC_STAGE_WP_LO: src = h->d_wp_lo; have = ff.Np * ff.Kw * 2; what = "Wp_lo"; break;
        case EVC_STAGE_ZT: src = h->d_zt; have = f.Mp * f.Ns * (int64_t)sizeof(float); what = "Zt"; break;
        case EVC_STAGE_XT: src = h->d_xt; have = t.Mp * t.Kp * 2; what = "Xt"; break;
        case EVC_STAGE_RT_HI: src = h->d_rt_hi; have = t.Np * t.Kp * 2; what = "Rt_hi"; break;
        case EVC_STAGE_RT_LO: src = h->d_rt_lo; have = t.Np * t.Kp * 2; what = "Rt_lo"; break;
        case EVC_STAGE_GD: src = h->d_Gd; have = t.planes * t.Mp * t.Np * (int64_t)sizeof(float); what = "Gd"; break;
        case EVC_STAGE_GH_PART:
            src = fused ? (const void *)h->d_gh_part3 : (const void *)h->d_gh_part2;
            have = (int64_t)h->g.L * (fused ? ff.ntile_part : f.ntiles_s) * h->g.S * (int64_t)sizeof(float);
            what = "gh_part";
            break;
        case EVC_STAGE_FX_PART:
            src = fused ? (const void *)h->d_fx_part3 : (const void *)h->d_fx_part2;
            have = (int64_t)h->g.L * (fused ? ff.ntile_part : f.ntiles_s) * (int64_t)sizeof(double);
            what = "fx_part";
            break;
        case EVC_STAGE_X: src = h->d_x1h; have = f.Xrows * f.Kw * 2; what = "the one-hot operand X"; break;
        default:
            set_error(name + ": unknown stage " + std::to_string(which) + " (EVC_STAGE_WT_HI .. EVC_STAGE_X)");
            return 1;
    }
    if (!src) {
        set_error(name + ": the handle has not allocated " + what + " (evc_plm_set_forward selects the buffers)");
        return 1;
    }
    if (bytes != have) {
        set_error(name + ": bytes must be the allocation of " + what + ", " + std::to_string(have));
        return 1;
    }
    EVC_CUDA(cudaSetDevice(h->device));
    EVC_CUDA(cudaDeviceSynchronize());
    EVC_CUDA(cudaMemcpy(dst, src, (size_t)bytes, cudaMemcpyDefault));
    return 0;
}

int evc_plm_copy_onehot(const evc_plm_t *h, void *host_dst, int64_t bytes)
{
    return copy_stage("evc_plm_copy_onehot", h, EVC_STAGE_X, host_dst, bytes);
}

int evc_plm_copy_stage(const evc_plm_t *h, int32_t which, void *dst, int64_t bytes)
{
    return copy_stage("evc_plm_copy_stage", h, which, dst, bytes);
}

int64_t evc_fit_workspace_bytes(int64_t n, int32_t m) { return n > 0 && m > 0 ? fit_work_bytes(n, m) : -1; }

int evc_fit_workspace_split_bytes(int64_t n, int32_t m, int32_t host_pairs, int64_t *device_bytes,
                                  int64_t *host_bytes)
{
    if (!device_bytes || !host_bytes) { set_error("evc_fit_workspace_split_bytes: null pointer"); return 1; }
    if (n <= 0 || m < 1 || m > 32 || host_pairs < 0 || host_pairs > m) {
        set_error("evc_fit_workspace_split_bytes: invalid arguments (need n >= 1, 1 <= m <= 32, "
                  "0 <= host_pairs <= m)");
        return 1;
    }
    fit_work_bytes(n, m, host_pairs, device_bytes, host_bytes);
    return 0;
}

int evc_plm_set_host_history(evc_plm_t *h, int32_t host_pairs)
{
    if (!h) { set_error("evc_plm_set_host_history: null handle"); return 1; }
    if (host_pairs < 0 || host_pairs > 32) {
        set_error("evc_plm_set_host_history: host_pairs must be in 0..32");
        return 1;
    }
    h->host_pairs = host_pairs;         // the next evc_plm_fit reallocates a workspace with another split
    return 0;
}

int evc_plm_host_bytes(const evc_plm_t *h, int64_t *bytes_out, double *pin_seconds_out)
{
    if (!h || !bytes_out) { set_error("evc_plm_host_bytes: null pointer"); return 1; }
    *bytes_out = fit_work_host_bytes(h->fit);
    if (pin_seconds_out) *pin_seconds_out = fit_work_pin_seconds(h->fit);
    return 0;
}

int evc_plm_set_profiling(evc_plm_t *h, int32_t enable)
{
    if (!h) { set_error("evc_plm_set_profiling: null handle"); return 1; }
    EVC_CUDA(cudaSetDevice(h->device));
    if (enable && !h->ev[0])
        for (int k = 0; k < 6; k++) EVC_CUDA(cudaEventCreate(&h->ev[k]));
    h->profiling = enable != 0;
    h->ev_valid = false;
    return 0;
}

int evc_plm_last_stage_ms(evc_plm_t *h, float *ms_out)
{
    if (!h || !ms_out) { set_error("evc_plm_last_stage_ms: null pointer"); return 1; }
    if (h->bwd_mode == 1 && h->tc.n_chunks > 1) {
        set_error("evc_plm_last_stage_ms: per-stage timing is not recorded when the sequences are processed in "
                  "chunks (evc_plm_set_seq_chunk); time the whole evaluation instead");
        return 1;
    }
    if (!h->ev_valid) { set_error("evc_plm_last_stage_ms: no profiled evaluation recorded"); return 1; }
    EVC_CUDA(cudaEventSynchronize(h->ev[5]));
    for (int k = 0; k < 5; k++) EVC_CUDA(cudaEventElapsedTime(&ms_out[k], h->ev[k], h->ev[k + 1]));
    return 0;
}

int evc_plm_add_regulariser(evc_plm_t *h, const float *d_x, float *d_g, double *d_fx, float lambda_h,
                            float lambda_J, void *stream)
{
    if (!h || !d_x || !d_g || !d_fx) { set_error("evc_plm_add_regulariser: null pointer"); return 1; }
    cudaStream_t st = as_stream(stream);
    double *partial = reduction_scratch(st);
    if (!partial) return 1;
    return regulariser(d_x, d_g, nullptr, h->g.n_params, (int64_t)h->g.L * h->g.q, lambda_h, lambda_J, d_fx, nullptr,
                       nullptr, d_fx + 1, nullptr, partial, st);
}

int evc_plm_eval_host(evc_plm_t *h, const float *x, float *gout, double *fx_out, float lambda_h,
                      float lambda_J)
{
    if (!h || !x || !gout || !fx_out) { set_error("evc_plm_eval_host: null pointer"); return 1; }
    EVC_CUDA(cudaSetDevice(h->device));
    const size_t nb = (size_t)h->g.n_params * sizeof(float);
    if (!h->d_x_tmp) {
        if (!dalloc(h, &h->d_x_tmp, nb) || !dalloc(h, &h->d_g_tmp, nb) || !dalloc(h, &h->d_fx_tmp, 2 * sizeof(double))) {
            set_error("evc_plm_eval_host: device allocation failed");
            return 1;
        }
    }
    EVC_CUDA(cudaMemcpyAsync(h->d_x_tmp, x, nb, cudaMemcpyHostToDevice, 0));
    if (evc_plm_eval_data(h, h->d_x_tmp, h->d_g_tmp, h->d_fx_tmp, nullptr)) return 1;
    if (evc_plm_add_regulariser(h, h->d_x_tmp, h->d_g_tmp, h->d_fx_tmp, lambda_h, lambda_J, nullptr)) return 1;
    EVC_CUDA(cudaMemcpyAsync(gout, h->d_g_tmp, nb, cudaMemcpyDeviceToHost, 0));
    EVC_CUDA(cudaMemcpyAsync(fx_out, h->d_fx_tmp, 2 * sizeof(double), cudaMemcpyDeviceToHost, 0));
    EVC_CUDA(cudaStreamSynchronize(0));
    return 0;
}

int evc_plm_weighted_counts(evc_plm_t *h, float *d_fi_counts, float *d_fij_counts, void *stream)
{
    if (!h || !d_fi_counts || !d_fij_counts) { set_error("evc_plm_weighted_counts: null pointer"); return 1; }
    cudaStream_t st = as_stream(stream);
    const PlmGeom &g = h->g;
    if (h->bwd_mode == 1 && h->d_gh_part2) {
        // tensor-core path: f_ij = Xt (w X)^T through the same backward product (weights as bf16 hi + lo), chunk by
        // chunk when the sequences are processed in chunks (Xt is then rebuilt for each)
        const int ntiles = h->tcf.ntiles_s;
        const PlmTcGeom &t = h->tc;
        for (int c = 0; c < t.n_chunks; c++) {
            const int64_t n0 = (int64_t)c * t.C, nreal = std::min(t.C, g.N - n0);
            if (t.n_chunks > 1 && plm_tc_build_xt(g, t, h->d_msa4, h->d_xt, n0, st)) return 1;
            if (plm_tc_onehot_residual(g, ntiles, h->d_msa4, h->d_wts, h->d_rt_hi, h->d_rt_lo, t.Kp, h->d_gh_part2,
                                       h->d_fx_part2, n0, nreal, st))
                return 1;
            if (plm_tc_backward(g, t, h->tc_maps, h->d_Gd, 0, c, st)) return 1;
        }
        if (plm_tc_finalize_pairs(g, t, h->d_Gd, t.planes, d_fij_counts, 0.5f, st)) return 1;
        return plm_finalize_fields_n(g, h->d_gh_part2, nullptr, d_fi_counts, nullptr, ntiles, st);
    }
    if (require_gather_q(h, "evc_plm_weighted_counts") || ensure_gather(h)) return 1;
    EVC_CUDA(cudaMemsetAsync(h->d_G, 0, (size_t)g.w_floats() * sizeof(float), st));
    if (plm_onehot_residual(g, h->d_msa4, h->d_wts, h->d_R, h->d_gh_part, st)) return 1;
    if (plm_backward(g, h->d_R, h->d_perm, h->d_bstart, h->d_G, st)) return 1;
    return plm_finalize(g, h->d_G, h->d_gh_part, nullptr, d_fi_counts, d_fij_counts, nullptr, 0.5f, st);
}

// ---- 8(f) rows f1 / f2 ------------------------------------------------------------------------------
int evc_ec_scores(const float *d_J_tri, const float *d_fij_tri, const float *d_fi, int32_t L, int32_t q,
                  float *d_fn_raw, float *d_fn_zero_sum, float *d_mi, void *stream)
{
    if (!d_J_tri) { set_error("evc_ec_scores: null pointer"); return 1; }
    return ec_scores(d_J_tri, d_fij_tri, d_fi, L, q, d_fn_raw, d_fn_zero_sum, d_mi, as_stream(stream));
}

int evc_plm_energies(evc_plm_t *h, const float *d_x, double *d_out, void *stream)
{
    if (!h || !d_x || !d_out) { set_error("evc_plm_energies: null pointer"); return 1; }
    cudaStream_t st = as_stream(stream);
    const PlmGeom &g = h->g;
    if (ensure_expanded(h)) return 1;          // no bucket lists: the energies take every supported q
    if (plm_expand(g, d_x, h->d_W, st)) return 1;
    // the residual buffer (L * Nr * S floats) is free outside an evaluation: reuse it for the per-site partials
    return plm_energies(g, h->d_W, d_x, h->d_msa4, h->d_R, d_out, st);
}

// ---- a8 vector algebra --------------------------------------------------------------------------
int evc_plm_pack_fx(const double *d_fx, float *d_limbs, void *stream)
{
    if (!d_fx || !d_limbs) { set_error("evc_plm_pack_fx: null pointer"); return 1; }
    return fx_pack(d_fx, d_limbs, as_stream(stream));
}
int evc_plm_unpack_fx(const float *d_limbs, double *d_fx, void *stream)
{
    if (!d_fx || !d_limbs) { set_error("evc_plm_unpack_fx: null pointer"); return 1; }
    return fx_unpack(d_limbs, d_fx, as_stream(stream));
}
int evc_vec_dot(const float *d_a, const float *d_b, int64_t n, double *d_out, void *stream)
{
    cudaStream_t st = as_stream(stream);
    double *partial = reduction_scratch(st);
    if (!partial) return 1;
    return vec_dot(d_a, d_b, n, d_out, partial, st);
}
int evc_vec_axpby(float *d_y, const float *d_x, float a, float b, int64_t n, void *stream)
{
    return vec_axpby(d_y, d_x, a, b, n, as_stream(stream));
}
int evc_vec_copy(float *d_dst, const float *d_src, int64_t n, void *stream)
{
    EVC_CUDA(cudaMemcpyAsync(d_dst, d_src, (size_t)n * sizeof(float), cudaMemcpyDeviceToDevice,
                             as_stream(stream)));
    return 0;
}
int evc_vec_sub(float *d_out, const float *d_a, const float *d_b, int64_t n, void *stream)
{
    return vec_sub(d_out, d_a, d_b, n, as_stream(stream));
}
int evc_vec_checksum(const float *d_v, int64_t n, uint64_t *d_out, void *stream)
{
    return vec_checksum(d_v, n, d_out, as_stream(stream));
}
int evc_lbfgs_direction(float *d_d, const float *d_g, const float *d_S, const float *d_Y, const double *d_ys,
                        double *d_scratch, int64_t n, int32_t m, int32_t bound, int32_t end, void *stream)
{
    if (bound > m || bound < 0 || m <= 0) { set_error("evc_lbfgs_direction: bad history bounds"); return 1; }
    cudaStream_t st = as_stream(stream);
    double *partial = reduction_scratch(st);
    if (!partial) return 1;
    std::vector<const float *> S(m), Y(m);
    for (int j = 0; j < m; j++) {
        S[j] = d_S + (int64_t)j * n;
        Y[j] = d_Y + (int64_t)j * n;
    }
    // d_scratch: [0] = y.y of the newest pair, [1] = the coefficient, [2 .. 2+m) = alpha
    return lbfgs_direction(d_d, d_g, S.data(), Y.data(), d_ys, d_scratch + 2, d_scratch + 1, d_scratch, n, m, bound,
                           end, partial, st);
}
int evc_lbfgs_update_pair(float *d_S_slot, float *d_Y_slot, const float *d_x, const float *d_xp,
                          const float *d_g, const float *d_gp, double *d_ys_slot, double *d_yy, int64_t n,
                          void *stream)
{
    cudaStream_t st = as_stream(stream);
    double *partial = reduction_scratch(st);
    if (!partial) return 1;
    return lbfgs_update_pair(d_S_slot, d_Y_slot, d_x, d_xp, d_g, d_gp, d_ys_slot, d_yy, n, partial, st);
}
int evc_fn_scores(const float *d_J_tri, int32_t L, int32_t q, float *d_fn, void *stream)
{
    return fn_scores(d_J_tri, L, q, d_fn, as_stream(stream));
}

}  // extern "C"
