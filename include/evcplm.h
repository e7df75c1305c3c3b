/*
 * libevcplm -- C ABI of the H100-native pseudo-likelihood Potts-model engine.
 *
 * This is the drop-in boundary for the ONE numerically heavy step of the
 * EVcouplings pipeline: what evcouplings/couplings/tools.py:126-307 (run_plmc)
 * obtains today by fork/exec of the external `plmc` C/OpenMP binary
 * (argv built at tools.py:202-262, subprocess at tools.py:266, caller
 * evcouplings/couplings/protocol.py:203-218).  The entry points below are
 * what a ctypes binding of that call site needs (INTEGRATION.md shows the
 * binding); evcouplings_b200/ is the Python host that mirrors run_plmc on top
 * of them.
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / C++ types.
 *   - "d_" arguments are device pointers on the handle's device, "h_"/unprefixed
 *     host pointers.  `stream` is a cudaStream_t passed as void* (NULL = default).
 *   - every function returns 0 on success, non-zero on failure;
 *     evc_last_error() gives the message (thread-local).
 *   - the caller owns all buffers it passes; the library owns what it allocates
 *     inside a handle until evc_plm_destroy.
 *   - a handle is not re-entrant; independent handles may be used from
 *     different threads or processes (one process per GPU for multi-GPU runs).  The
 *     evc_vec_*, evc_lbfgs_*, evc_plm_add_regulariser and evc_hamming_* entry points keep
 *     their small reduction / candidate scratch per (device, stream) inside the library:
 *     concurrent callers must use different streams (or different devices).
 *
 * Parameter vector layout (identical to the plmc_v2 .model file read by
 * evcouplings/couplings/model.py:354-389):
 *     x = [ h : L*q floats | J : L(L-1)/2 blocks of q*q floats,
 *           pairs (i<j) in row-major (i,j) order, block[a][b], a = state at i ]
 * Sequence codes: uint8, 0..q-1 = model states; with gap_code >= 0 (plmc -g,
 * "ignore_gaps") the value gap_code (== q) marks a gap: the site is skipped as
 * a conditional and contributes nothing as a neighbour.
 * Alphabet sizes: evc_plm_create / evc_plm_tc_bytes take q in {4, 5, 20, 21}
 * (protein and nucleotide, with or without the gap state), as they always
 * have.  evc_plm_create_alphabet / evc_plm_tc_bytes_alphabet take every
 * alphabet whose codes fit the 5 bit-planes of the Hamming pass (codes < 32):
 * 2 <= q <= 32 with the gap as a state, 2 <= q <= 31 with gap_code == q.
 * The tensor-core path, the pair counts and the energies take the whole range;
 * the gather objective kernels (forward / backward mode 0) exist for q in
 * {4, 5, 20, 21} only and return an error naming evc_plm_set_forward(h, 1)
 * for any other q, including evc_plm_eval_data / evc_plm_weighted_counts on a
 * handle left at the gather defaults.
 */
#ifndef EVCPLM_H
#define EVCPLM_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EVCPLM_ABI_VERSION 2

typedef struct evc_plm evc_plm_t;

/* ---- library / device -------------------------------------------------- */
int evc_abi_version(void);
const char *evc_last_error(void);
int evc_device_count(void);                  /* <0 on error                */
int evc_device_info(int32_t device, int32_t *sm_count, int32_t *cc_major, int32_t *cc_minor,
                    int64_t *total_mem_bytes);

/* ---- (b) O(N^2 L) pairwise-Hamming sequence reweighting ------------------
 * Replaces plmc's reweighting pass (stderr "Effective number of samples",
 * parsed at tools.py:55) and the in-tree twin
 * evcouplings/align/alignment.py:1192-1233 (num_cluster_members).
 * counts[s] = #{ t : #(codes[s,k] == codes[t,k]) >= min_identical }, self
 * included, gap == gap counts as identical.  min_identical is the integer form
 * of "pair_id / L >= theta" (alignment.py:1229), computed by the host.
 * Codes must be < 32 (5 bit-planes): evc_hamming_counts rejects larger ones
 * on the host; evc_hamming_pack takes device codes and does not check them.
 */
int evc_hamming_counts(const uint8_t *codes, int64_t N, int32_t L, int32_t min_identical,
                       int32_t device, int32_t *counts_out);

/* device-resident building blocks (multi-GPU: each rank counts a tile range,
 * the host all-reduces the int32 counters) */
int64_t evc_hamming_plane_words(int64_t N, int32_t L);   /* uint32 words of the bit-plane buffer */
int64_t evc_hamming_num_tiles(int64_t N);                /* upper-triangular 128x128 pair tiles   */
int evc_hamming_pack(const uint8_t *d_codes, int64_t N, int32_t L, uint32_t *d_planes, void *stream);
int evc_hamming_count_tiles(const uint32_t *d_planes, int64_t N, int32_t L, int32_t min_identical,
                            int64_t tile_begin, int64_t tile_end, int32_t *d_counts /* += */,
                            void *stream);

/* The same counts over distinct rows with multiplicities (evc_msa_unique): a pair of neighbours (s, t) credits
 * mult[t] to s and mult[s] to t instead of 1, so counts[u] = sum_v mult[v] [id(u, v) >= min_identical], u itself
 * included -- the count every copy of u gets from evc_hamming_counts on the full rows.  Same pruning, tiles and
 * hooks; the counters stay int32, so the multiplicities must sum to less than 2^31 (the host entry point checks
 * that they are >= 1 and do). */
int evc_hamming_counts_mult(const uint8_t *codes, const int32_t *mult, int64_t N, int32_t L, int32_t min_identical,
                            int32_t device, int32_t *counts_out);
int evc_hamming_count_tiles_mult(const uint32_t *d_planes, const int32_t *d_mult, int64_t N, int32_t L,
                                 int32_t min_identical, int64_t tile_begin, int64_t tile_end,
                                 int32_t *d_counts /* += */, void *stream);

/* ---- distinct rows of the code matrix ---------------------------------------------------------------------
 * Rows merge only if all L codes are equal (a 64-bit row hash, a stable radix sort by hash, then an exact byte
 * comparison inside each hash group: a hash collision never merges distinct rows).  The result does not depend on
 * the launch or the stream.  With U distinct rows:
 *   d_first[0..U)   the first row of each distinct row, ascending (the identity when there are no repeats)
 *   d_inverse[0..N) row -> distinct index
 *   d_mult[0..U)    multiplicities (sum N)
 * d_first and d_mult must hold N entries (U is known only at the end); *U_out is a host pointer, and the call
 * synchronises `stream` to fill it.  Scratch: about 40 bytes per row, allocated and freed stream-ordered on `stream`.
 * N < 2^31. */
int evc_msa_unique(const uint8_t *d_codes /* N x L */, int64_t N, int32_t L, int32_t *d_first, int32_t *d_inverse,
                   int32_t *d_mult, int64_t *U_out, void *stream);
/* host-buffer convenience of evc_msa_unique (first_out and mult_out hold N entries; the first U are written) */
int evc_msa_unique_host(const uint8_t *codes /* N x L */, int64_t N, int32_t L, int32_t device, int32_t *first_out,
                        int32_t *inverse_out, int32_t *mult_out, int64_t *U_out);

/* f3 twin of identities_to_seq (evcouplings/align/alignment.py:1156-1189): d_out[n] = #{k : codes[n,k] == seq[k]} */
int evc_identities_to_seq(const uint8_t *d_codes /* N x L */, const uint8_t *d_seq /* L */, int64_t N, int32_t L,
                          int32_t *d_out, void *stream);

/* ---- f4: compiled A2M / FASTA ingest (host code) ---------------------------------------------------------
 * Replaces the reference's in-tree text readers (evcouplings/align/alignment.py:42-74 read_fasta, 410-443
 * sequences_to_matrix, 479-495 map_matrix) and plmc's own parser (8a row a4).  Return 0 ok, 1 I/O or argument
 * error, 2 malformed alignment (no sequences / zero length / ragged rows); message in evc_last_error().
 *   evc_a2m_scan:   number of records, common row width, bytes for the NUL-separated record ids
 *   evc_a2m_read:   raw characters (n_rows x width, as in the file: case and '.' preserved) and the ids
 *   evc_msa_encode: codes_out[v][k] = lut[raw[row_v][cols[k]]] for the VALID rows only (a row is valid iff no
 *                   character of the whole row maps to 255), valid_out[r] in {0,1}, *n_valid_out rows written */
int evc_a2m_scan(const char *path, int64_t *n_rows, int64_t *width, int64_t *ids_bytes);
int evc_a2m_read(const char *path, int64_t n_rows, int64_t width, uint8_t *raw, char *ids, int64_t ids_bytes);
int evc_msa_encode(const uint8_t *raw, int64_t n_rows, int64_t width, const uint8_t *lut, const int64_t *cols,
                   int64_t n_cols, uint8_t *valid_out, uint8_t *codes_out, int64_t *n_valid_out);

/* ---- (a) PLM objective + gradient -----------------------------------------
 * Replaces plmc's negative-log-posterior evaluation (the inner loop of its
 * L-BFGS; SURVEY.md 8a row a7).
 */
/* fails before any device work for q outside {4, 5, 20, 21} or a code out of range */
int evc_plm_create(evc_plm_t **out, const uint8_t *codes /* host, N x L */, int64_t N, int32_t L,
                   int32_t q, int32_t gap_code /* -1: gap is a model state */,
                   const float *weights /* host, N */, int32_t device);
/* evc_plm_create for any alphabet size above (2 <= q <= 32; q <= 31 with gap_code == q); the same handle */
int evc_plm_create_alphabet(evc_plm_t **out, const uint8_t *codes /* host, N x L */, int64_t N, int32_t L,
                            int32_t q, int32_t gap_code /* -1: gap is a model state */,
                            const float *weights /* host, N */, int32_t device);
void evc_plm_destroy(evc_plm_t *h);
int64_t evc_plm_num_params(const evc_plm_t *h);          /* L*q + L(L-1)/2*q*q */

/* data term on this handle's sequences:  d_g[0..n) = d/dx of
 * -sum_s w_s sum_i log P(s_i | s_-i),  d_fx[0] = that sum (double).
 * No regulariser (so shards can be summed with one all-reduce). */
int evc_plm_eval_data(evc_plm_t *h, const float *d_x, float *d_g, double *d_fx, void *stream);

/* Backward implementation of the data term: 0 = gather/bucket kernel (shared-memory bound, default),
 * 1 = dense one-hot contraction on the Hopper tensor cores (wgmma; bf16 hi/lo split of the residuals, fp32
 * accumulation in registers).  Both produce the same gradient within fp32 tolerance; bench.py reports both. */
int evc_plm_set_backward(evc_plm_t *h, int32_t mode);
/* Forward implementation: 0 = gather kernel (fp32 couplings streamed through shared memory),
 * 1 = logits as a wgmma GEMM (couplings split in bf16 hi + lo, fp32 accumulation) followed by a
 * softmax/residual kernel; 2 = the same GEMM with softmax / residuals fused into its epilogue (no logits
 * matrix in HBM; protein alphabets, falls back to 1 otherwise).  Modes 1 and 2 imply the tensor-core backward. */
int evc_plm_set_forward(evc_plm_t *h, int32_t mode);

/* Arithmetic of the tensor-core products (SURVEY.md 8b `precision`; BASELINE configs[4] "bf16 tiles / fp32
 * parameters"): 0 (default) = fp32-equivalent: the real-valued operand (couplings forward, residuals backward)
 * enters as TWO bf16 terms hi + lo (16 mantissa bits), two wgmma per K slice; 1 = bf16 tiles: ONE bf16
 * term, one wgmma per K slice (half the tensor-core work).  Parameters, accumulation (registers, K chunks
 * promoted with fp32 round-to-nearest adds), softmax and the optimiser stay fp32 in both modes.  No effect on
 * the gather kernels.  May be changed between evaluations. */
int evc_plm_set_precision(evc_plm_t *h, int32_t mode);

/* Sequences per chunk of the tensor-core path (0 = the whole shard, the default).  The sequence-indexed operands
 * of the tensor-core path (one-hot X and Xt, logits Zt, residuals Rt_hi / Rt_lo: about 12 N L q bytes) are then
 * sized for seq_chunk sequences, rounded up to a multiple of 768, and every evaluation streams the shard through
 * them: the couplings operand is expanded once, then each chunk builds its one-hot operands and runs the logits
 * GEMM, the softmax and the backward GEMM, which adds into the gradient planes; the finalizes run once.  The
 * objective and g_h are bit-identical to the unchunked evaluation (same per-tile partial sums in the same order);
 * g_J and the pair counts differ by the summation order of the backward product only.  seq_chunk >= N is one
 * chunk, i.e. the unchunked path.  Call it before evc_plm_set_backward / evc_plm_set_forward: it fails if the
 * tensor-core buffers already exist for another chunk size.  With more than one chunk the fused forward (mode 2)
 * falls back to mode 1, the gather forward is refused by evc_plm_eval_data, and the gather kernels (backward
 * mode 0, evc_plm_energies) are not chunked. */
int evc_plm_set_seq_chunk(evc_plm_t *h, int64_t seq_chunk);
/* Device bytes a handle with these parameters allocates on the default tensor-core path (evc_plm_create, then
 * evc_plm_set_seq_chunk(seq_chunk), evc_plm_set_forward(1)); computed on the host from the same geometry as the
 * allocations (no device needed; sm_count picks the split of the backward product). */
int evc_plm_tc_bytes(int64_t N, int32_t L, int32_t q, int32_t gap_code, int64_t seq_chunk, int32_t sm_count,
                     int64_t *bytes_out);
/* the same count for a handle of evc_plm_create_alphabet (any alphabet size above) */
int evc_plm_tc_bytes_alphabet(int64_t N, int32_t L, int32_t q, int32_t gap_code, int64_t seq_chunk,
                              int32_t sm_count, int64_t *bytes_out);
/* Device bytes the handle holds now, including the L-BFGS workspace once evc_plm_fit has allocated it. */
int64_t evc_plm_device_bytes(const evc_plm_t *h);
/* Copies the handle's one-hot operand of the tensor-core forward (Xrows * Kw * 2 bytes, Xrows = the sequences of a
 * chunk rounded up to 384, Kw = L*q rounded up to 64; `bytes` must equal that) to host memory, in the form the
 * selected forward reads: 2:4-sparse fragments for evc_plm_set_forward(1), dense bf16 rows for 2.  With sequence
 * chunks it holds the last chunk evaluated.  For tests; synchronises the device.  Same as
 * evc_plm_copy_stage(h, EVC_STAGE_X, ...). */
int evc_plm_copy_onehot(const evc_plm_t *h, void *host_dst, int64_t bytes);
/* Intermediate buffers of the tensor-core evaluation, for evc_plm_copy_stage.  Layouts (row-major, Lq = L*q; Mp, Np,
 * Kw, Kp, Ns as in plm_tc_geometry / plm_tcf_geometry, Np' = ceil(L / 8) * 176 of the fused forward):
 *   WT_HI, WT_LO  bf16 [Mp][Kw]   couplings of the sparse forward, row (i,a), column (j,b)
 *   WP_HI, WP_LO  bf16 [Np'][Kw]  couplings of the fused forward, rows in 88-row halves of 4 sites x 21 + 4 zero rows
 *   ZT            fp32 [Mp][Ns]   logits without h, column = sequence of the chunk
 *   XT            bf16 [Mp][Kp]   one-hot operand of the backward product, row (j,b), column = sequence of the chunk
 *   RT_HI, RT_LO  bf16 [Np][Kp]   residuals (or weights, for the counts), row (i,a), column = sequence of the chunk
 *   GD            fp32 [planes][Mp][Np]  K slices of the backward product, row (j,b), column (i,a)
 *   GH_PART       fp32 [L][tiles][S]     per-tile partial sums of g_h / f_i of the selected forward
 *   FX_PART       fp64 [L][tiles]        per-tile partial sums of -loglk of the selected forward
 *   X             the one-hot operand of the forward (evc_plm_copy_onehot) */
#define EVC_STAGE_WT_HI 0
#define EVC_STAGE_WT_LO 1
#define EVC_STAGE_WP_HI 2
#define EVC_STAGE_WP_LO 3
#define EVC_STAGE_ZT 4
#define EVC_STAGE_XT 5
#define EVC_STAGE_RT_HI 6
#define EVC_STAGE_RT_LO 7
#define EVC_STAGE_GD 8
#define EVC_STAGE_GH_PART 9
#define EVC_STAGE_FX_PART 10
#define EVC_STAGE_X 11
/* Copies the whole of one of these buffers (`bytes` must equal its allocation) to `dst`, host or device memory
 * (cudaMemcpyDefault).  Fails, naming the reason, for an unknown `which` and for a buffer the handle has not
 * allocated.  With sequence chunks the per-chunk buffers hold the last chunk evaluated.  For tests; synchronises
 * the device. */
int evc_plm_copy_stage(const evc_plm_t *h, int32_t which, void *dst, int64_t bytes);
/* Device bytes of the workspace evc_plm_fit allocates for n parameters and history m (host function). */
int64_t evc_fit_workspace_bytes(int64_t n, int32_t m);
/* Correction pairs of the L-BFGS history kept in pinned host memory (0, the default, .. m of the fit).  Each such
 * pair moves two n-vectors (about 8 n bytes) out of device memory: the fit's device workspace
 * is (5 + 2 (m - host_pairs)) vectors, and host_pairs x 2 vectors are allocated with cudaHostAlloc(Mapped) when the
 * next evc_plm_fit creates its workspace.  The two-loop recursion and the pair update then read and write those
 * slots over PCIe with the same kernels, so the iterates are bit-identical to a device-resident history; each
 * iteration streams about 4 host_pairs vectors across the link.  evc_plm_fit fails if host_pairs exceeds its
 * history m.  Call it before evc_plm_fit; a later call takes effect with the next fit. */
int evc_plm_set_host_history(evc_plm_t *h, int32_t host_pairs);
/* Device and pinned host bytes of the evc_plm_fit workspace for n parameters, history m and host_pairs pairs in
 * host memory (host function; host_pairs = 0 gives device_bytes = evc_fit_workspace_bytes(n, m), host_bytes = 0). */
int evc_fit_workspace_split_bytes(int64_t n, int32_t m, int32_t host_pairs, int64_t *device_bytes,
                                  int64_t *host_bytes);
/* Pinned host bytes the handle holds now (the host-resident correction pairs once evc_plm_fit has allocated them)
 * and the seconds that allocation took (pin_seconds_out may be NULL).  evc_plm_device_bytes counts only the
 * device part of the fit workspace. */
int evc_plm_host_bytes(const evc_plm_t *h, int64_t *bytes_out, double *pin_seconds_out);

/* Per-stage device timing of the LAST evc_plm_eval_data call (CUDA events recorded on the stream the
 * kernels were launched on): ms_out[5] = {expand (+ clear), forward (gather kernel or logits GEMM),
 * softmax kernel (0 on the gather forward), backward kernel, finalize}.
 * Used by bench.py to report the dominant kernel's roofline live.  Not recorded when the evaluation runs in
 * sequence chunks (evc_plm_set_seq_chunk): evc_plm_last_stage_ms then returns an error. */
int evc_plm_set_profiling(evc_plm_t *h, int32_t enable);
int evc_plm_last_stage_ms(evc_plm_t *h, float *ms_out);

/* d_g += 2*lambda*x (lambda_h on the first L*q entries, lambda_J on the rest);
 * d_fx[1] = d_fx[0] + lambda_h*|h|^2 + lambda_J*|J|^2   (d_fx[0] = -loglk kept) */
int evc_plm_add_regulariser(evc_plm_t *h, const float *d_x, float *d_g, double *d_fx,
                            float lambda_h, float lambda_J, void *stream);

/* host-buffer convenience (H2D of x, evaluation, D2H of g inside the call):
 * fx_out[0] = -loglk, fx_out[1] = full objective. */
int evc_plm_eval_host(evc_plm_t *h, const float *x, float *g, double *fx_out,
                      float lambda_h, float lambda_J);

/* ---- a6: weighted single / pair counts for the .model file ---------------
 * d_fi_counts[L*q], d_fij_counts[L(L-1)/2*q*q] (tri blocks [a][b]) receive
 * sum_s w_s [s_i=a] and sum_s w_s [s_i=a][s_j=b]; the host normalises
 * (N_eff, or per-site / per-pair non-gap weight under ignore_gaps). */
int evc_plm_weighted_counts(evc_plm_t *h, float *d_fi_counts, float *d_fij_counts, void *stream);

/* ---- a8: the whole L-BFGS fit on the device (replaces plmc's libLBFGS loop; iteration cap = plmc `-m`,
 * evcouplings/couplings/tools.py:226-228) ---------------------------------------------------------------
 * Minimises  -sum_s w_s sum_i log P(s_i | s_-i) + lambda_h |h|^2 + lambda_J |J|^2  from the start point in d_x
 * (device, n floats; overwritten with the result).  All vectors live in the handle; the host sees six doubles
 * per objective evaluation.  Status codes carry libLBFGS's names (plmc prints them after
 * "Gradient optimization:", parsed at tools.py:57). */
enum {
    EVC_LBFGS_SUCCESS = 0,
    EVC_LBFGS_ALREADY_MINIMIZED = 2,
    EVC_LBFGSERR_CANCELED = -1021,
    EVC_LBFGSERR_INVALIDPARAMETERS = -1000,
    EVC_LBFGSERR_MINIMUMSTEP = -1001,
    EVC_LBFGSERR_MAXIMUMSTEP = -1002,
    EVC_LBFGSERR_MAXIMUMLINESEARCH = -1003,
    EVC_LBFGSERR_MAXIMUMITERATION = -1004,
    EVC_LBFGSERR_WIDTHTOOSMALL = -1005,
    EVC_LBFGSERR_ROUNDING_ERROR = -1006,
    EVC_LBFGSERR_INCREASEGRADIENT = -1007
};
typedef struct {
    int32_t max_iterations;      /* 0 = until convergence                                             */
    int32_t m;                   /* correction pairs kept (1..32)                                      */
    float epsilon;               /* stop when |g| / max(1, |x|) <= epsilon                             */
    float lambda_h, lambda_J;
    int32_t max_linesearch;
    double min_step, max_step, ftol, gtol, xtol;
    int32_t precision_schedule;  /* 0: keep the handle's precision; 1: bf16 tiles until
                                    |g|/max(1,|x|) <= switch_factor * epsilon (or the line search fails),
                                    then fp32-equivalent products to the end                            */
    float switch_factor;
} evc_fit_params_t;
typedef struct {
    int32_t status;              /* EVC_LBFGS*                                                          */
    int32_t iterations;
    int32_t evaluations;
    int32_t switched_at;         /* iteration at which precision_schedule 1 left the bf16 mode, or -1   */
    double fx, negloglk;
    double seconds;
} evc_fit_result_t;
/* Sum d_buf[0..count) over all ranks in place, asynchronously on `stream` (NCCL all-reduce in the Python host).
 * The buffer is the gradient followed by 4 floats that carry -loglk as exact fixed-point limbs: ONE collective
 * per evaluation.  NULL = single rank.  Return non-zero to abort. */
typedef int (*evc_allreduce_cb)(void *user, float *d_buf, int64_t count, void *stream);
/* Called once per iteration (the row of plmc's iteration table, tools.py:59-83); non-zero return cancels. */
typedef int (*evc_progress_cb)(void *user, int32_t iteration, double fx, double xnorm, double gnorm, double step,
                               int32_t linesearch_evals, double negloglk, double hnorm, double enorm);
void evc_fit_default_params(evc_fit_params_t *p);
int evc_plm_fit(evc_plm_t *h, float *d_x, const evc_fit_params_t *params, evc_allreduce_cb allreduce,
                void *allreduce_user, evc_progress_cb progress, void *progress_user, evc_fit_result_t *result,
                void *stream);

/* ---- checkpoint / resume of evc_plm_fit ---------------------------------------------------------------------
 * The fit's state at an iteration boundary, i.e. right after iteration k's progress callback.  The n-vectors are not
 * in the struct: evc_plm_fit_vector gives their addresses (x and g of the accepted iterate, and the S / Y slots of
 * the correction pairs by ring index).  The `hist` newest pairs sit at ring slots (end - hist .. end - 1) mod m.
 * The pair of iteration k (s = x_k - x_{k-1}, y = g_k - g_{k-1}) is already stored when the state is taken: the
 * fit performs that update before the callback, which is what the continued loop would do next, so no x_{k-1} or
 * g_{k-1} is needed and a run stopped at its iteration cap can be continued to a higher cap.  Continuing from the
 * state (evc_plm_fit_checkpointed with `resume`) replays what the uninterrupted loop does after that callback: the
 * convergence test, the cap test, the bf16 -> hi+lo switch of precision_schedule 1, the direction and the step,
 * and gives bit-identical iterates when the objective's summation order is the same (same ranks, same sequence
 * chunk; host-resident pairs never change bits). */
#define EVC_FIT_STATE_VERSION 1
typedef struct {
    int32_t version;             /* EVC_FIT_STATE_VERSION                                                   */
    int32_t returning;           /* 1: the fit returns right after this call, with `status`; 0: interval    */
    int32_t status;              /* EVC_LBFGS* status the fit returns with (0 when `returning` is 0)        */
    int32_t k;                   /* iterations completed (the last row of the iteration table)             */
    int32_t evaluations;         /* objective evaluations so far                                           */
    int32_t m, hist, end;        /* history size, stored pairs, ring slot written next                     */
    int32_t low;                 /* 1: precision_schedule 1 is still in its bf16 phase                      */
    int32_t switched_at;         /* as evc_fit_result_t                                                     */
    int64_t n;                   /* parameters                                                              */
    double fx, negloglk, xnorm, gnorm;
    double ys[32];               /* y.s per ring slot                                                       */
    double yy;                   /* y.y of the newest pair                                                  */
    double seconds;              /* fit seconds so far (continued by a resumed fit)                         */
} evc_fit_state_t;
/* Called at an iteration boundary once `checkpoint_interval` seconds have passed since the fit started or since the
 * last call (every boundary for 0; never for a negative interval), when the progress callback cancels, and when the
 * fit returns with a consistent state (EVC_LBFGS_SUCCESS, EVC_LBFGSERR_MAXIMUMITERATION or a line-search failure,
 * which returns the last accepted point); `returning` tells the last call apart.  The vectors are valid through
 * evc_plm_fit_vector until the callback returns; copy them on `stream`.  Non-zero return aborts the fit. */
typedef int (*evc_checkpoint_cb)(void *user, const evc_fit_state_t *state, void *stream);
/* evc_plm_fit plus checkpoints.  With `resume` (a state a callback was given, for the same problem and params.m),
 * the start point in d_x is ignored: the fit continues from the workspace, which the host filled between
 * evc_plm_fit_prepare and this call, and the result still lands in d_x.  evaluations, iterations and seconds of the
 * result count from the start of the first fit. */
int evc_plm_fit_checkpointed(evc_plm_t *h, float *d_x, const evc_fit_params_t *params, evc_allreduce_cb allreduce,
                             void *allreduce_user, evc_progress_cb progress, void *progress_user,
                             evc_checkpoint_cb checkpoint, void *checkpoint_user, double checkpoint_interval,
                             const evc_fit_state_t *resume, evc_fit_result_t *result, void *stream);
/* Allocate (or keep) the fit workspace for history m and the handle's host pairs, so that the host can fill it
 * before a resuming evc_plm_fit_checkpointed with the same m. */
int evc_plm_fit_prepare(evc_plm_t *h, int32_t m);
/* Address of one n-vector of the fit workspace: which = EVC_FIT_VEC_X / _G (the accepted iterate), or _S / _Y with
 * `slot` the ring index 0..m-1.  Device memory, or the device address of mapped pinned host memory for the slots
 * m - host_pairs .. m - 1 (evc_plm_set_host_history; the same address on the host under unified addressing).  Valid
 * inside the checkpoint callback and between evc_plm_fit_prepare and the resuming call. */
enum { EVC_FIT_VEC_X = 0, EVC_FIT_VEC_G = 1, EVC_FIT_VEC_S = 2, EVC_FIT_VEC_Y = 3 };
int evc_plm_fit_vector(evc_plm_t *h, int32_t which, int32_t slot, float **ptr_out);

/* -loglk <-> 4 floats appended to the gradient (three exact fixed-point limbs, resolution 2^-16, |fx| < 1.3e11, up to 64 ranks):
 * a data-parallel evaluation then needs ONE all-reduce of n + 4 floats (SURVEY.md 8e `[fx, g]`).
 * Each limb is a float holding an integer: 0 <= limb0, limb1 < 2^18, |limb2| < 2^17 (the sign lives there), so float32
 * sums over up to 64 ranks are exact in any order, and the decoded value is sum_r round_half_even(fx_r * 2^16) / 2^16.
 * The 4th float is 0 for a value in that range.  A -loglk that is NaN, infinite or at least 9e15 / 2^16 (1.373e11) in
 * magnitude is not carried as a finite number: evc_plm_pack_fx sets the 4th float to NaN, which survives the sum, and
 * evc_plm_unpack_fx gives NaN whenever the 4th float is not 0, so every rank sees NaN as a single rank would. */
int evc_plm_pack_fx(const double *d_fx, float *d_limbs, void *stream);
int evc_plm_unpack_fx(const float *d_limbs, double *d_fx, void *stream);

/* ---- a8: on-device L-BFGS vector algebra ----------------------------------
 * All scalars stay on the device (double); the host reads back only what the
 * line search needs. */
int evc_vec_dot(const float *d_a, const float *d_b, int64_t n, double *d_out, void *stream);
int evc_vec_axpby(float *d_y, const float *d_x, float a, float b, int64_t n, void *stream); /* y = a*x + b*y */
int evc_vec_copy(float *d_dst, const float *d_src, int64_t n, void *stream);
int evc_vec_sub(float *d_out, const float *d_a, const float *d_b, int64_t n, void *stream);
/* Exact, order-independent checksum of the float bit patterns b_i of d_v[0..n):
 *     d_out[0] = sum_i mix(i, b_i) mod 2^64,  mix(i, b) = splitmix64_finalizer((i + 1) * 0x9E3779B97F4A7C15 ^ b)
 * with 64-bit indices (splitmix64's finalizer: z ^= z >> 30; z *= 0xBF58476D1CE4E5B9; z ^= z >> 27;
 * z *= 0x94D049BB133111EB; z ^= z >> 31).  d_v may be the device address of mapped pinned host memory. */
int evc_vec_checksum(const float *d_v, int64_t n, uint64_t *d_out, void *stream);
/* two-loop recursion: d = -H g using `bound` stored pairs ending before slot
 * `end` (ring of m); d_S/d_Y are m x n row-major; d_ys[m] holds y.s per slot;
 * d_scratch needs m + 2 doubles. */
int evc_lbfgs_direction(float *d_d, const float *d_g, const float *d_S, const float *d_Y,
                        const double *d_ys, double *d_scratch, int64_t n, int32_t m,
                        int32_t bound, int32_t end, void *stream);
/* s = x - xp, y = g - gp into slot, d_ys[slot] = y.s, d_scratch[0] = y.y (fused) */
int evc_lbfgs_update_pair(float *d_S_slot, float *d_Y_slot, const float *d_x, const float *d_xp,
                          const float *d_g, const float *d_gp, double *d_ys_slot, double *d_yy,
                          int64_t n, void *stream);

/* ---- SURVEY 8(f) "next" rows ------------------------------------------------
 * f1: per-pair scores of CouplingsModel._calculate_ecs (evcouplings/couplings/model.py:777-827):
 *     Frobenius norm of each J_ij block in the raw gauge (plmc's _ECs.txt) and in the zero-sum gauge
 *     (model.py:179-233), and mutual information from f_ij / f_i (d_fij_tri / d_fi / d_mi may be NULL).
 *     The APC (model.py:744-775) is an L x L host operation.
 * f2: statistical energies of this handle's sequences under parameters x (model.py:25-60 _hamiltonians):
 *     d_out[n][3] = {H, H_J, H_h} (double). */
int evc_ec_scores(const float *d_J_tri, const float *d_fij_tri, const float *d_fi, int32_t L, int32_t q,
                  float *d_fn_raw, float *d_fn_zero_sum, float *d_mi, void *stream);
int evc_plm_energies(evc_plm_t *h, const float *d_x, double *d_out, void *stream);

/* ---- a10: EC scores (Frobenius norm of each J block, raw gauge) ---------- */
int evc_fn_scores(const float *d_J_tri, int32_t L, int32_t q, float *d_fn /* L(L-1)/2 */, void *stream);

/* ---- Gibbs sampling of the fitted model ---------------------------------------------------------------------
 * Target: P(s) ~ exp(beta H(s)), H(s) = sum_i h_i(s_i) + sum_{i<j} J_ij(s_i, s_j) (the energy of evc_plm_energies:
 * larger H is more probable), codes 0..q-1, 2 <= q <= 32.  A model fitted with ignored gaps has q states and no gap,
 * so its samples contain none.
 * Update: systematic-scan heat bath.  A sweep visits i = 0..L-1 in order and redraws s_i from softmax_a(beta Z_i(a)),
 * Z_i(a) = h_i(a) + sum_{j != i} J_ij(a, s_j) (the logits of the PLM forward).
 * Draw: v_a = beta Z_i(a) in fp32, m = max v, p_a = exp(v_a - m), c_a the inclusive prefix sum over a = 0..q-1 (fp32);
 * s_i = the smallest a with u c_{q-1} < c_a, or q-1 if none.  u has 25 significant bits, so u and u c_{q-1} are
 * formed in double, where they are exact.
 * Randomness is counter-based: chain c's trajectory depends only on x, its start, seed, its global index
 * c = chain_offset + local index, the sweeps run and beta -- not on n_chains, the launch, how the sweeps are split over
 * calls, or the device.  With mix = splitmix64's finaliser (as in evc_vec_checksum), phi = 0x9E3779B97F4A7C15:
 *     key(c)     = mix(seed ^ mix((c + 1) phi))
 *     u(c, t, i) = ((mix(key(c) + k phi) >> 40) + 0.5) 2^-24,  k = (t L + i + 1) mod 2^64
 * t is the global sweep index, counted from 0 at evc_sampler_create; t = -1 is the uniform start, s_i = floor(u q).
 * Fields: each chain keeps Z (L q fp32); when s_i changes from a to b, Z += U[(i,b), :] - U[(i,a), :], U the full
 * symmetric coupling matrix ((L q)^2 fp32, zero diagonal blocks; 70.6 MB at L = 200, q = 21), built on the device at
 * create.  Before every sweep t with t % EVC_SAMPLER_REFRESH == 0 (t = 0 included) Z is recomputed from s in fp32,
 * h_i(a) first, then j ascending; refreshing at global sweep indices keeps split runs bit-identical.
 * Limits: one chain's Z row and codes (4 L q + L bytes, rounded up to 16) must fit one CTA's 227 KB of shared memory:
 * L q up to about 58 000 (L about 2 700 at q = 21).  Device memory: U plus 4 L q + L bytes per chain.
 *   evc_sampler_create: d_x = the model in the layout above (device, n floats); init = host n_chains x L codes < q, or
 *                       NULL for the uniform start.  q, L, n_chains, chain_offset, the init codes and null pointers are
 *                       checked before any device work.  Synchronises the device.
 *   evc_sampler_run:    `sweeps` sweeps at inverse temperature beta, asynchronously on `stream`; changes_out (host,
 *                       may be NULL; if given the call synchronises `stream`) receives the number of site changes.
 *   evc_sampler_codes:  copies the current codes (n_chains x L uint8, device) on `stream`. */
#define EVC_SAMPLER_REFRESH 32
typedef struct evc_sampler evc_sampler_t;
int evc_sampler_create(evc_sampler_t **out, const float *d_x /* L*q + L(L-1)/2*q*q */, int32_t L, int32_t q,
                       const uint8_t *init /* host, n_chains x L codes < q; NULL = uniform start */,
                       int64_t n_chains, int64_t chain_offset, uint64_t seed, int32_t device);
int evc_sampler_run(evc_sampler_t *s, int32_t sweeps, float beta, int64_t *changes_out /* site changes, may be NULL */,
                    void *stream);
int evc_sampler_codes(const evc_sampler_t *s, uint8_t *d_codes_out /* n_chains x L */, void *stream);
void evc_sampler_destroy(evc_sampler_t *s);
/* evc_sampler_set_model: on `stream`, loads new parameters d_x (same L, q; device, n floats) into a live sampler:
 * copies h and rebuilds U.  The chains' codes, counters and sweep index are kept; the next sweep, whatever its index,
 * recomputes Z from the codes first, and the refreshes at t % EVC_SAMPLER_REFRESH == 0 continue as before.  A
 * sampler that never calls it runs exactly as above.  d_x is read on `stream` and may be freed once it has run. */
int evc_sampler_set_model(evc_sampler_t *s, const float *d_x, void *stream);
/* evc_sampler_anneal: annealed importance sampling (AIS) along p_beta(s) ~ exp(sum_i h_i(s_i) + beta H_J(s)),
 * H_J(s) = sum_{i<j} J_ij(s_i, s_j): beta scales the couplings only, so beta = 0 is the independent-site model.
 * Runs K sweeps at the handle's global sweep indices t, t + 1, ..., t + K - 1 with the counters, the refresh rule
 * (t % EVC_SAMPLER_REFRESH) and the Z of evc_sampler_run.  Before sweep k = 1..K, once any refresh due at that sweep
 * has run, every chain c
 *     forms H_J = 1/2 sum_i (Z_i(s_i) - h_i(s_i)), each difference and the sum in double, in a fixed lane and
 *           butterfly order (exact when Z is: see the sampler's fields above),
 *     adds  d_logw[c] += ((double)betas[k] - (double)betas[k-1]) H_J   (double, no contraction),
 * and then sweeps at beta_k = betas[k] with the draw above applied to v_a = h_i(a) + beta_k (Z_i(a) - h_i(a)) in fp32,
 * each operation rounded on its own (no contraction).  betas (host, K + 1 finite values) and K >= 0 are checked
 * before any device work; the handle copies the schedule to the device on `stream`, so betas may be freed on return.
 * d_logw (device, n_chains doubles) accumulates: it is read and written on `stream`, never reset.  A chain's
 * trajectory and weight depend only on x, its start, seed, its global index, the sweeps and the schedule, so a
 * schedule split over calls (betas[0..a], then betas[a..K]) gives the bits of one call, and handles over disjoint
 * chain_offset ranges give the weights of one handle.  changes_out as in evc_sampler_run.
 * Estimator (model_ops.log_partition): every chain is first drawn exactly from p_0 by one sweep at beta = 0 (betas =
 * {0, 0}), then annealed along beta_k = k / K; log Z = log Z_0 + logsumexp_c(log w_c) - log M, with log Z_0 =
 * sum_i log sum_a exp h_i(a). */
int evc_sampler_anneal(evc_sampler_t *s, const float *betas /* host, K + 1 */, int32_t K,
                       double *d_logw /* device, n_chains, accumulated */, int64_t *changes_out, void *stream);
/* evc_sampler_create_conditional: a sampler whose chains redraw only the free sites F = free_sites[0] < free_sites[1]
 * < ... < free_sites[nf-1], each from its allowed states, while the clamped sites C (every other site) keep each
 * chain's start codes, its context x_c.  The free sites of chain c follow the Potts model with couplings J_FF and
 * per-chain fields
 *     hc_c,k(a) = h_{F_k}(a) + sum_{j in C} J_{F_k j}(a, x_c,j)   (fp32, h first, then j ascending, each add rounded
 *                                                                  on its own; J read at 64-bit offsets of x)
 * folded once at create (n_chains x nf q floats, evc_sampler_conditional_fields copies them out).  The chain is the
 * one above over the free sites only:
 *   fields:   Z over (k, a) of the free sites; before every sweep t with t % EVC_SAMPLER_REFRESH == 0, Z = hc_c, then
 *             + U_FF[(k', s_k'), :] for free k' ascending, U_FF = U restricted to F ((nf q)^2 fp32, zero diagonal
 *             blocks; the full U is never built); a change a -> b of free site k adds U_FF[(k,b), :] - U_FF[(k,a), :];
 *             Z persists between calls;
 *   counters: u(c, t, F_k) with the model's L, so a free site's uniforms do not depend on which other sites are
 *             clamped;
 *   draw:     with mask allowed[k] (bit a = state a allowed), v_a = beta Z_k(a) on allowed lanes and -inf elsewhere,
 *             m = the max over the allowed lanes, p_a = exp(v_a - m) (0 when disallowed), c_a the inclusive prefix
 *             sum; s = the smallest a with u c_{q-1} < c_a, or, if none, the highest allowed state.  With every mask
 *             full this is the draw above.
 * With nf = L and full masks, hc = h and U_FF = U bit for bit and the refresh order is the plain one, so every chain
 * gives exactly the codes of evc_sampler_create's handle for the same x, start, seed, chain_offset, beta and sweeps.
 * Start: init (host n_chains x L codes < q; required when nf < L), or the uniform start when nf = L and init is NULL.
 * A free site may start outside its mask; every sweep redraws every free site, so after one sweep every free site
 * holds an allowed state.  allowed: host, nf masks, each non-zero with no bit >= q; NULL = all q states.
 * Checked before any device work, as in evc_sampler_create, with: 1 <= nf <= L; free_sites strictly ascending in
 * [0, L); the masks; init given when nf < L; one chain's row over the free sites, 4 nf q + nf bytes rounded up to 16,
 * plus the CTA's table of free sites and masks, 8 nf bytes rounded up to 16, within one CTA's 227 KB (nf q up to
 * about 58 000, whatever L).  Device memory: U_FF plus 8 nf q + L bytes per chain
 * (Z, hc, codes).  Synchronises the device.
 * On a conditional handle evc_sampler_run sweeps the free sites; evc_sampler_codes returns full n_chains x L rows, the
 * clamped sites always holding init; evc_sampler_anneal and evc_sampler_set_model return 1 and do no device work.
 *   evc_sampler_conditional_fields: copies hc (n_chains x nf q floats, device, [c][k q + a]) on `stream`; returns 1
 *                                   on a handle that is not conditional. */
int evc_sampler_create_conditional(evc_sampler_t **out, const float *d_x, int32_t L, int32_t q,
                                   const int32_t *free_sites /* host, nf strictly ascending */, int32_t nf,
                                   const uint32_t *allowed /* host, nf masks; NULL = all q states */,
                                   const uint8_t *init /* host n_chains x L, required when nf < L */,
                                   int64_t n_chains, int64_t chain_offset, uint64_t seed, int32_t device);
int evc_sampler_conditional_fields(const evc_sampler_t *s, float *d_hc_out /* n_chains x nf q */, void *stream);
/* Replica exchange (parallel tempering) on a plain or conditional handle.
 * Ladder: R >= 2 inverse temperatures 0 <= beta_0 < beta_1 < ... < beta_{R-1}, finite fp32.  A handle of n_chains =
 * G R chains holds G ladders: ladder l is the chains l R .. l R + R - 1, its global index g = chain_offset / R + l
 * (chain_offset a multiple of R).  At evc_sampler_set_ladder chain l R + k holds rung k.
 * Sweeps: every chain runs the sweep of evc_sampler_run (or of the conditional handle) at the beta of the rung it
 * holds, v_a = beta_c Z_i(a): the counters u(c, t, i), the start, Z and its refresh rule are unchanged.  So a ladder
 * whose betas are all equal gives exactly the codes of evc_sampler_run at that beta, bit for bit.
 * Energy: after the last sweep before each swap round every chain forms, from its Z, in double,
 *     H = sum_i h_i(s_i) + 1/2 sum_i (Z_i(s_i) - h_i(s_i)),
 * each difference and each sum rounded on its own in the lane and butterfly order of evc_sampler_anneal's H_J (lane l
 * of a warp sums the sites l, l + 32, ... ascending, then xor-butterfly over offsets 16, 8, 4, 2, 1; both sums, then
 * sum_h + 0.5 sum_J).  On a conditional handle: hc_c in place of h, over the free sites only.
 * Swaps: a swap round n follows every global sweep t with (t + 1) % swap_interval == 0, n = (t + 1) / swap_interval
 * - 1.  Round n visits the pairs (k, k + 1) with k = n mod 2, n mod 2 + 2, ... < R - 1 in ascending k (the
 * deterministic even-odd scheme of non-reversible tempering).  With x the chain at beta_k and y the chain at
 * beta_{k+1}, Delta = ((double)beta_{k+1} - (double)beta_k) (H(x) - H(y)) in double, no contraction, and the swap is
 * accepted if Delta >= 0 or u < exp(Delta), with
 *     swap_key(g)  = key(2^63 + g)   (key of the sampler's counters; no chain index reaches 2^63, and every step of key
 *                                     is a bijection, so no chain's stream is reused)
 *     u(g, n, k)   = ((mix(swap_key(g) + k' phi) >> 40) + 0.5) 2^-24,  k' = (n R + k + 1) mod 2^64.
 * An accepted swap exchanges the rung labels (betas) of the two chains, not their codes: each chain keeps its Z, its
 * codes and its counters.  A ladder's trajectory depends only on x, its starts, seed, g, the sweeps, the ladder and
 * swap_interval: not on how the sweeps are split over calls (also between swap rounds), on G or on the device.
 * Round trips: a chain that reaches rung R-1 after rung 0 and then rung 0 again completes one; they are counted per
 * ladder after every round (the chain at rung 0 at set_ladder counts as having visited rung 0).
 *   evc_sampler_set_ladder: betas (host, R values) and swap_interval >= 1; R, the betas, n_chains % R, chain_offset % R
 *                           and swap_interval are checked before any device work.  A ladder is set once: setting the
 *                           same ladder again does nothing, a different one returns 1.  On a conditional handle with
 *                           clamped sites every chain of a ladder must hold the same clamped codes (checked on the
 *                           device's codes).  Synchronises the device.  Once a ladder is set, evc_sampler_anneal and
 *                           evc_sampler_set_model return 1; evc_sampler_run stays legal (all chains at its beta,
 *                           advancing t; the swap rounds of the sweeps it runs do not happen).
 *   evc_sampler_temper:     `sweeps` tempered sweeps with their swap rounds, asynchronously on `stream`.  d_swaps
 *                           (device, 2 (R - 1) int64, may be NULL) accumulates, never reset: [k] += the attempted swaps
 *                           of pair (k, k + 1), [R - 1 + k] += the accepted ones, over the handle's ladders (exact
 *                           integer sums, so the sums of handles over disjoint ladders add up to one handle's).
 *                           changes_out as in evc_sampler_run.
 *   evc_sampler_ladder_state: copies on `stream`, each output may be NULL: d_rung (n_chains int32, the rung each chain
 *                           holds), d_energy (n_chains double, H of the last swap round, 0 before the first) and
 *                           d_round_trips (n_chains / R int64, per ladder). */
int evc_sampler_set_ladder(evc_sampler_t *s, const float *betas /* host, R */, int32_t R, int64_t swap_interval);
int evc_sampler_temper(evc_sampler_t *s, int32_t sweeps, int64_t *d_swaps /* device, 2 (R - 1), accumulated */,
                       int64_t *changes_out, void *stream);
int evc_sampler_ladder_state(const evc_sampler_t *s, int32_t *d_rung /* n_chains */,
                             double *d_energy /* n_chains */, int64_t *d_round_trips /* n_chains / R */, void *stream);
/* Design: the highest-scoring states of a plain, conditional or tempered handle.
 * Record: once evc_sampler_record_best has run, every sweep t of evc_sampler_run and evc_sampler_temper ends, for
 * every chain c, by forming H from the chain's Z exactly as the tempered energy above (lane and butterfly order; on a
 * conditional handle hc_c and the free sites, so H is the conditional energy) and, if H > best_energy[c] strictly,
 * storing best_energy[c] = H, best_codes[c] = the chain's codes (full rows of L codes, clamped sites included) and
 * best_sweep[c] = t.  The record starts at -inf with best_sweep = -1, so the first recorded sweep always sets it, and a
 * NaN H is never recorded.  It lives on the device and persists across calls, so a run split over calls gives the
 * record of one call.  Recording reads the chain only: codes, Z and changes are those of the same calls without it.
 * Descent: evc_sampler_descend runs `sweeps` zero-temperature sweeps at the handle's global sweep indices, with the
 * refresh rule (t % EVC_SAMPLER_REFRESH, and the sweep after evc_sampler_set_model) and the change update of the
 * handle's sweep.  Site i (a free site on a conditional handle) visits the allowed states A_i (the mask; every a < q on
 * a plain handle) and takes m = max_{a in A_i} Z_i(a) in fp32; s_i stays if s_i is in A_i and Z_i(s_i) == m, else
 * becomes the smallest a in A_i with Z_i(a) == m (if none, as when Z holds a NaN, s_i stays).  No uniforms are drawn,
 * beta and the rungs of a ladder play no part, and every chain runs every sweep (a later refresh may re-round Z and
 * move a chain that had stopped).  The descent advances t and leaves the record as it is.
 *   evc_sampler_record_best: starts (or restarts) the record on `stream`: best_energy = -inf, best_sweep = -1 and
 *                            best_codes = the current codes.  Device memory: 16 + L bytes per chain.
 *   evc_sampler_best:        copies the record on `stream`, each output may be NULL: d_energy (n_chains double),
 *                            d_codes (n_chains x L uint8), d_sweep (n_chains int64).  Returns 1 before any record.
 *   evc_sampler_descend:     asynchronously on `stream`; d_settled (device, n_chains uint8, may be NULL) receives 1
 *                            for a chain whose last sweep of the call changed no site, else 0 (not written when
 *                            sweeps = 0); changes_out as in evc_sampler_run.  sweeps < 0 returns 1.
 * evc_sampler_anneal on a recording handle returns 1 and does no device work. */
int evc_sampler_record_best(evc_sampler_t *s, void *stream);
int evc_sampler_best(const evc_sampler_t *s, double *d_energy /* n_chains */, uint8_t *d_codes /* n_chains x L */,
                     int64_t *d_sweep /* n_chains */, void *stream);
int evc_sampler_descend(evc_sampler_t *s, int32_t sweeps, uint8_t *d_settled /* n_chains, may be NULL */,
                        int64_t *changes_out, void *stream);

/* ---- Boltzmann-machine learning (bmDCA) ----------------------------------------------------------------------
 * Refines x so that the model's one- and two-site marginals match target statistics f (same layout as x:
 * [f_i | f_ij tri blocks], as stored in a .model).  Objective, the full-likelihood counterpart of the PLM one,
 * divided by N_eff:
 *     F(theta) = -sum_k theta_k f_k + log Z(theta) + lambda'_h |h|^2 + lambda'_J |J|^2,
 *     lambda'_h = lambda_h / n_eff, lambda'_J = lambda_J / n_eff (from the .model header; n_eff <= 0 only with both
 *     lambda zero, then lambda' = 0).
 * F is strictly convex when lambda' > 0, so its optimum is unique and no gauge needs fixing.  One update with M
 * persistent chains and learning rate eta (model_ops.BoltzmannLearner drives it):
 *     1. S sweeps of every chain at beta = 1 (evc_sampler_run);
 *     2. c = exact counts of the chains' codes in x layout (evc_code_counts);
 *     3. for every k, in double, each operation rounded on its own (no FMA):
 *            g_k = (c_k / M - f_k) + lam2 theta_k,  lam2 = 2 lambda'_h (k < L q) or 2 lambda'_J,
 *            theta_k <- fp32_rn(theta_k - eta g_k)     (evc_bm_update);
 *     4. load theta into the sampler (evc_sampler_set_model).
 * Given the model, seed, M, S, burn-in sweeps, eta and the number of updates the result is bit-identical, however
 * the updates are split over calls.  Limits: those of the sampler (L q up to about 58 000).
 *   evc_code_counts: exact integer counts of N device rows of codes (< q, not checked, as in evc_hamming_pack), on
 *                    `stream`: site counts [i q + a], then for pairs i < j in row-major order [pair][a][b]; n =
 *                    L q + L(L-1)/2 q q counters.  Every counter is written exactly once with a plain store (no
 *                    memset, no global atomics), so the result does not depend on the launch.  2 <= q <= 32,
 *                    1 <= L <= 32768, 1 <= N <= 2^31 - 1.  Work N L(L+1)/2 shared-memory increments; HBM bytes
 *                    N L codes read (re-read from L2 by every CTA), 4 n counts written.
 *   evc_bm_update:   step 3 on `stream`, fused over all n parameters (x in place; Lq = L q fields first).
 *                    d_stats[0], [1] (device doubles) receive max |c/M - f| over the fields and over the couplings
 *                    (order-independent maxima, so deterministic).  About 16 n bytes of HBM traffic.
 * Several ranks (model_ops.BoltzmannLearner over a process group): rank r runs the chains [lo, hi) of the M global ones
 * as a sampler with chain_offset = lo and N = hi - lo, and counts them with evc_code_counts.  The counts of disjoint
 * chain ranges are summed as integers (exact and order-independent while M < 2^31) before the update, and the sum
 * equals the counts of one handle over all M chains; every rank then calls evc_bm_update with the global M, so every
 * rank holds the x of one process, bit for bit. */
int evc_code_counts(const uint8_t *d_codes, int64_t N, int32_t L, int32_t q, uint32_t *d_counts /* n */,
                    void *stream);
int evc_bm_update(float *d_x, const uint32_t *d_counts, int64_t M, const float *d_f, int64_t n, int32_t Lq,
                  double eta, double lam2_h, double lam2_J, double *d_stats /* 2 */, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* EVCPLM_H */
