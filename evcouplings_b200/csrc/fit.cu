// a8: the L-BFGS driver of the PLM fit, resident on the device (SURVEY.md 8a row a8, 8b `evc_plm_fit`).
//
// plmc minimises the objective with libLBFGS on the host CPU (reference call site
// evcouplings/couplings/tools.py:226-228 passes the iteration cap `-m`).  Here every n-vector (x, g, search
// direction, m correction pairs) lives in HBM inside the handle, except the correction pairs that
// evc_plm_set_host_history moves to pinned host memory; per objective evaluation the host sees six
// doubles (one 48-byte D2H + one stream synchronisation) -- the scalars the More-Thuente line search decides on.
//
//   trial point      x_try = x + t d                                    (vec_step)
//   objective        evc_plm_eval_data (expand -> GEMM -> softmax -> GEMM -> symmetrise)
//   multi-rank       -loglk is packed as three exact fixed-point limbs behind the gradient so that ONE
//                    all-reduce (callback; NCCL in the Python host) carries [g, fx]; every partial sum of a
//                    limb is an integer < 2^24, i.e. the fp32 reduction is exact and order-independent
//   regulariser      g += 2 lambda x fused with the five reductions of the scalar block   (regulariser)
//   two-loop         d = -H g with alpha and the coefficients kept on the device        (lbfgs_direction)
// The vector kernels are those of vecops.cu: fixed grid, fixed tree => every rank of a data-parallel run takes
// bit-identical decisions without broadcasting anything.
//
// The line search is the safeguarded cubic/quadratic interpolation of More & Thuente (1994) with libLBFGS's
// default constants (ftol 1e-4, gtol 0.9, xtol 1e-7, 40 trials), first step 1/|g|, then 1.
#include <chrono>
#include <cmath>
#include <cstring>

#include "../../include/evcplm.h"
#include "common.cuh"
#include "internal.h"

namespace evc {

// device scalar block (doubles); SC_DG .. SC_XXJ are the regulariser's four dots in its order
enum { SC_FX = 0, SC_NLL, SC_DG, SC_GG, SC_XXH, SC_XXJ, SC_YY, SC_COEF, SC_YS = 8 /* [m] */, SC_ALPHA = 8 + 32 /* [m] */, SC_COUNT = 8 + 64 };

// ---- host-side line search (More & Thuente) ---------------------------------------------------------
struct MtState {
    double x, fx, dx, y, fy, dy;
    bool brackt;
};

static double cubic_min(double u, double fu, double du, double v, double fv, double dv)
{
    const double d = v - u;
    const double theta = (fu - fv) * 3.0 / d + du + dv;
    const double s = std::max(std::fabs(theta), std::max(std::fabs(du), std::fabs(dv)));
    const double a = theta / s;
    double gamma = s * std::sqrt(std::max(0.0, a * a - (du / s) * (dv / s)));
    if (v < u) gamma = -gamma;
    const double p = gamma - du + theta;
    const double q = gamma - du + gamma + dv;
    return u + (p / q) * d;
}

static double cubic_min2(double u, double fu, double du, double v, double fv, double dv, double xmin, double xmax)
{
    const double d = v - u;
    const double theta = (fu - fv) * 3.0 / d + du + dv;
    const double s = std::max(std::fabs(theta), std::max(std::fabs(du), std::fabs(dv)));
    const double a = theta / s;
    double gamma = s * std::sqrt(std::max(0.0, a * a - (du / s) * (dv / s)));
    if (u < v) gamma = -gamma;
    const double p = gamma - dv + theta;
    const double q = gamma - dv + gamma + du;
    const double r = p / q;
    if (r < 0.0 && gamma != 0.0) return v - r * d;
    if (a < 0) return xmax;
    return xmin;
}

static double quad_min(double u, double fu, double du, double v, double fv)
{
    const double a = v - u;
    return u + du / ((fu - fv) / a + du) / 2.0 * a;
}

static double quad_min2(double u, double du, double v, double dv)
{
    const double a = u - v;
    return v + dv / (dv - du) * a;
}

// safeguarded trial-value update (More & Thuente sec. 4); returns true on an inconsistent interval
static bool update_trial_interval(MtState &st, double &t, double ft, double dt, double tmin, double tmax)
{
    double x = st.x, fx = st.fx, dx = st.dx, y = st.y, fy = st.fy, dy = st.dy;
    bool brackt = st.brackt;
    const bool dsign = dx != 0.0 ? (dt * (dx / std::fabs(dx)) < 0.0) : (dt < 0.0);
    if (brackt) {
        if (t <= std::min(x, y) || std::max(x, y) <= t) return true;
        if (0.0 <= dx * (t - x)) return true;
        if (tmax < tmin) return true;
    }
    bool bound;
    double newt;
    if (fx < ft) {
        brackt = true;
        bound = true;
        const double mc = cubic_min(x, fx, dx, t, ft, dt), mq = quad_min(x, fx, dx, t, ft);
        newt = std::fabs(mc - x) < std::fabs(mq - x) ? mc : mc + 0.5 * (mq - mc);
    } else if (dsign) {
        brackt = true;
        bound = false;
        const double mc = cubic_min(x, fx, dx, t, ft, dt), mq = quad_min2(x, dx, t, dt);
        newt = std::fabs(mc - t) > std::fabs(mq - t) ? mc : mq;
    } else if (std::fabs(dt) < std::fabs(dx)) {
        bound = true;
        const double mc = cubic_min2(x, fx, dx, t, ft, dt, tmin, tmax), mq = quad_min2(x, dx, t, dt);
        if (brackt) newt = std::fabs(t - mc) < std::fabs(t - mq) ? mc : mq;
        else newt = std::fabs(t - mc) > std::fabs(t - mq) ? mc : mq;
    } else {
        bound = false;
        if (brackt) newt = cubic_min(t, ft, dt, y, fy, dy);
        else if (x < t) newt = tmax;
        else newt = tmin;
    }
    if (fx < ft) {
        y = t; fy = ft; dy = dt;
    } else {
        if (dsign) { y = x; fy = fx; dy = dx; }
        x = t; fx = ft; dx = dt;
    }
    newt = std::min(tmax, std::max(tmin, newt));
    if (brackt && bound) {
        const double mq = x + 0.66 * (y - x);
        if (x < y) { if (mq < newt) newt = mq; }
        else { if (newt < mq) newt = mq; }
    }
    st.x = x; st.fx = fx; st.dx = dx; st.y = y; st.fy = fy; st.dy = dy; st.brackt = brackt;
    t = newt;
    return false;
}

// ---- the fit workspace (owned by the handle) -----------------------------------------------------------
// The S / Y ring has m slots.  Slots m - host_pairs .. m - 1 live in mapped (zero-copy) pinned host memory owned by
// the workspace; the kernels read and write them over PCIe through their device addresses.  The two-loop recursion
// and the pair update touch each history vector as one sequential stream with no reuse inside an iteration, so the
// kernels and their arithmetic are the same for both kinds of slot and the iterates are bit-identical to a fully
// device-resident history.
struct FitWork {
    int64_t n = 0, stride = 0;
    int m = 0;
    int host_pairs = 0;
    float *x[2] = {nullptr, nullptr};   // current / trial parameters (ping-pong)
    float *g[2] = {nullptr, nullptr};   // gradients, each with 4 trailing floats for the packed -loglk
    float *d = nullptr;
    float *S = nullptr, *Y = nullptr;   // (m - host_pairs) x stride, device
    float *h_hist = nullptr;            // 2 host_pairs x stride, pinned host: the S slots, then the Y slots
    float *hist_dev = nullptr;          // device address of h_hist
    float *s[32] = {}, *y[32] = {};     // address of ring slot j: in S / Y, or in hist_dev for the last host_pairs
    double pin_seconds = 0.0;           // time taken to allocate and pin h_hist
    double *sc = nullptr;               // device scalars (SC_*)
    double *partial = nullptr;          // RED_PARTIALS
    double *fx_data = nullptr;          // [2] data-term -loglk written by evc_plm_eval_data
    double *h_sc = nullptr;             // pinned host copy of sc[0..8)
    int cur = 0;                        // x[cur], g[cur]: the accepted iterate (evc_plm_fit_vector)
};

void fit_work_free(FitWork *w)
{
    if (!w) return;
    for (int k = 0; k < 2; k++) { cudaFree(w->x[k]); cudaFree(w->g[k]); }
    cudaFree(w->d); cudaFree(w->S); cudaFree(w->Y); cudaFree(w->sc); cudaFree(w->partial); cudaFree(w->fx_data);
    if (w->h_sc) cudaFreeHost(w->h_sc);
    if (w->h_hist) cudaFreeHost(w->h_hist);
    delete w;
}

// device: x[2], g[2], d and the device slots of the S / Y ring, each of `stride` floats, plus the device scalars;
// host: the host slots of the ring (two vectors per pair)
void fit_work_bytes(int64_t n, int m, int host_pairs, int64_t *device_bytes, int64_t *host_bytes)
{
    const int64_t vb = round_up(n + 4, 64) * (int64_t)sizeof(float);
    *device_bytes = (5 + 2 * (int64_t)(m - host_pairs)) * vb +
                    (int64_t)(SC_COUNT + RED_PARTIALS + 2) * (int64_t)sizeof(double);
    *host_bytes = 2 * (int64_t)host_pairs * vb;
}
int64_t fit_work_bytes(int64_t n, int m)
{
    int64_t dev, host;
    fit_work_bytes(n, m, 0, &dev, &host);
    return dev;
}
int64_t fit_work_bytes(const FitWork *w)
{
    if (!w) return 0;
    int64_t dev, host;
    fit_work_bytes(w->n, w->m, w->host_pairs, &dev, &host);
    return dev;
}
int64_t fit_work_host_bytes(const FitWork *w)
{
    if (!w) return 0;
    int64_t dev, host;
    fit_work_bytes(w->n, w->m, w->host_pairs, &dev, &host);
    return host;
}
double fit_work_pin_seconds(const FitWork *w) { return w ? w->pin_seconds : 0.0; }

static FitWork *fit_work_create(int64_t n, int m, int host_pairs)
{
    FitWork *w = new (std::nothrow) FitWork();
    if (!w) return nullptr;
    w->n = n;
    w->m = m;
    w->host_pairs = host_pairs;
    w->stride = round_up(n + 4, 64);
    const size_t vb = (size_t)w->stride * sizeof(float);
    const int dev_pairs = m - host_pairs;
    bool ok = true;
    for (int k = 0; k < 2 && ok; k++)
        ok = cudaMalloc(&w->x[k], vb) == cudaSuccess && cudaMalloc(&w->g[k], vb) == cudaSuccess;
    ok = ok && cudaMalloc(&w->d, vb) == cudaSuccess &&
         (dev_pairs == 0 || (cudaMalloc(&w->S, vb * dev_pairs) == cudaSuccess &&
                             cudaMalloc(&w->Y, vb * dev_pairs) == cudaSuccess)) &&
         cudaMalloc(&w->sc, SC_COUNT * sizeof(double)) == cudaSuccess &&
         cudaMalloc(&w->partial, RED_PARTIALS * sizeof(double)) == cudaSuccess &&
         cudaMalloc(&w->fx_data, 2 * sizeof(double)) == cudaSuccess &&
         cudaMallocHost(&w->h_sc, 8 * sizeof(double)) == cudaSuccess;
    if (ok && host_pairs > 0) {
        const auto t0 = std::chrono::steady_clock::now();
        ok = cudaHostAlloc(&w->h_hist, vb * 2 * host_pairs, cudaHostAllocMapped) == cudaSuccess &&
             cudaHostGetDevicePointer(&w->hist_dev, w->h_hist, 0) == cudaSuccess;
        w->pin_seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    }
    if (!ok) {
        set_error(std::string("evc_plm_fit: workspace allocation failed: ") + cudaGetErrorString(cudaGetLastError()));
        fit_work_free(w);
        return nullptr;
    }
    for (int j = 0; j < m; j++) {
        const int64_t off = (int64_t)j * w->stride, host_off = (int64_t)(j - dev_pairs) * w->stride;
        w->s[j] = j < dev_pairs ? w->S + off : w->hist_dev + host_off;
        w->y[j] = j < dev_pairs ? w->Y + off : w->hist_dev + (int64_t)host_pairs * w->stride + host_off;
    }
    cudaMemset(w->sc, 0, SC_COUNT * sizeof(double));
    return w;
}

struct FitCtx {
    evc_plm_t *h;
    FitWork *w;
    const evc_fit_params_t *p;
    evc_allreduce_cb ar;
    void *ar_user;
    cudaStream_t st;
    int evals = 0;
};

// objective + gradient at w->x[which] into w->g[which]; dvec (may be null) gives g.d.  Host scalars in w->h_sc.
static int fit_evaluate(FitCtx &c, int which, const float *dvec)
{
    FitWork *w = c.w;
    float *x = w->x[which], *g = w->g[which];
    if (evc_plm_eval_data(c.h, x, g, w->fx_data, c.st)) return 1;
    const float *limbs = nullptr;
    if (c.ar) {
        if (fx_pack(w->fx_data, g + w->n, c.st)) return 1;
        if (c.ar(c.ar_user, g, w->n + 4, c.st)) { set_error("evc_plm_fit: all-reduce callback failed"); return 1; }
        limbs = g + w->n;
    }
    const int64_t nh = (int64_t)c.h->g.L * c.h->g.q;
    if (regulariser(x, g, dvec, w->n, nh, c.p->lambda_h, c.p->lambda_J, w->fx_data, limbs, w->sc + SC_NLL,
                    w->sc + SC_FX, w->sc + SC_DG, w->partial, c.st))
        return 1;
    EVC_CUDA(cudaMemcpyAsync(w->h_sc, w->sc, 8 * sizeof(double), cudaMemcpyDeviceToHost, c.st));
    EVC_CUDA(cudaStreamSynchronize(c.st));
    c.evals++;
    return 0;
}

// d = -H g by the two-loop recursion over the `bound` newest pairs (ring of m, `end` = next slot to write)
static int fit_direction(FitCtx &c, int cur, int bound, int end)
{
    FitWork *w = c.w;
    return lbfgs_direction(w->d, w->g[cur], w->s, w->y, w->sc + SC_YS, w->sc + SC_ALPHA, w->sc + SC_COEF,
                           w->sc + SC_YY, w->n, w->m, bound, end, w->partial, c.st);
}

// The fit loop behind evc_plm_fit and evc_plm_fit_checkpointed.  Without a checkpoint callback it launches exactly
// the kernels evc_plm_fit always launched, in the same order.
static int fit_run(evc_plm_t *h, float *d_x, const evc_fit_params_t *p, evc_allreduce_cb allreduce,
                   void *allreduce_user, evc_progress_cb progress, void *progress_user, evc_checkpoint_cb ckpt,
                   void *ckpt_user, double ckpt_interval, const evc_fit_state_t *resume, evc_fit_result_t *res,
                   void *stream)
{
    if (!h || !d_x || !p || !res) { set_error("evc_plm_fit: null pointer"); return 1; }
    if (p->m < 1 || p->m > 32) { set_error("evc_plm_fit: history m must be in 1..32"); return 1; }
    const int64_t n = evc_plm_num_params(h);
    EVC_CUDA(cudaSetDevice(h->device));
    if (h->host_pairs > p->m) {
        set_error("evc_plm_fit: " + std::to_string(h->host_pairs) + " host-resident correction pairs exceed the "
                  "history m = " + std::to_string(p->m) + " (evc_plm_set_host_history)");
        return 1;
    }
    if (resume) {
        if (resume->version != EVC_FIT_STATE_VERSION || resume->m != p->m || resume->n != n || resume->k < 0 ||
            resume->hist < 0 || resume->hist > resume->m || resume->end < 0 || resume->end >= resume->m ||
            resume->evaluations < 1) {
            set_error("evc_plm_fit_checkpointed: the resume state does not match this problem (version " +
                      std::to_string(resume->version) + ", m = " + std::to_string(resume->m) + ", n = " +
                      std::to_string(resume->n) + "; expected version " + std::to_string(EVC_FIT_STATE_VERSION) +
                      ", m = " + std::to_string(p->m) + ", n = " + std::to_string(n) + ")");
            return 1;
        }
        if (!h->fit || h->fit->m != p->m || h->fit->host_pairs != h->host_pairs) {
            set_error("evc_plm_fit_checkpointed: resuming needs the workspace filled after evc_plm_fit_prepare(h, m)");
            return 1;
        }
    }
    if (h->fit && (h->fit->m != p->m || h->fit->host_pairs != h->host_pairs)) {
        fit_work_free(h->fit);
        h->fit = nullptr;
    }
    if (!h->fit) h->fit = fit_work_create(n, p->m, h->host_pairs);
    FitWork *w = h->fit;
    if (!w) return 1;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    FitCtx c{h, w, p, allreduce, allreduce_user, st};
    const auto t_begin = std::chrono::steady_clock::now();
    auto t_saved = t_begin;
    const double t_offset = resume ? resume->seconds : 0.0;
    auto elapsed = [&](std::chrono::steady_clock::time_point since) {
        return std::chrono::duration<double>(std::chrono::steady_clock::now() - since).count();
    };
    const size_t nb = (size_t)n * sizeof(float);
    int &cur = w->cur;
    int k = 0, switched_at = -1;
    bool low = false;
    double fx = 0.0, nll = 0.0, xnorm = 0.0, gnorm = 0.0;
    auto finish = [&](int stat) {
        res->status = stat;
        res->iterations = k;
        res->evaluations = c.evals;
        res->switched_at = switched_at;
        res->fx = fx;
        res->negloglk = nll;
        res->seconds = t_offset + elapsed(t_begin);
        if (cudaMemcpyAsync(d_x, w->x[cur], nb, cudaMemcpyDeviceToDevice, st) != cudaSuccess ||
            cudaStreamSynchronize(st) != cudaSuccess) {
            set_error("evc_plm_fit: copying the result failed");
            return 1;
        }
        return 0;
    };
    int hist = 0, end = 0;
    double step = 0.0;
    // The correction pair of the iteration just accepted: s = x[cur] - x[prev], y = g[cur] - g[prev] into slot `end`
    // (device or pinned host memory).  `pair_pending` while it is owed; a checkpoint stores it before the state.
    bool pair_pending = false;
    auto add_pair = [&]() -> int {
        const int prev = cur ^ 1;
        if (lbfgs_update_pair(w->s[end], w->y[end], w->x[cur], w->x[prev], w->g[cur], w->g[prev], w->sc + SC_YS + end,
                              w->sc + SC_YY, n, w->partial, st))
            return 1;
        hist = std::min(p->m, hist + 1);
        end = (end + 1) % p->m;
        pair_pending = false;
        return 0;
    };
    // hand the state to the checkpoint callback; `returning`: the fit returns `status` right after
    auto save = [&](bool returning, int status) -> int {
        if (!ckpt) return 0;
        if (pair_pending && add_pair()) return 1;
        double sc[2 + 32];        // SC_YY, SC_COEF, SC_YS[0..m)
        EVC_CUDA(cudaMemcpyAsync(sc, w->sc + SC_YY, (2 + p->m) * sizeof(double), cudaMemcpyDeviceToHost, st));
        EVC_CUDA(cudaStreamSynchronize(st));
        evc_fit_state_t s;
        memset(&s, 0, sizeof(s));
        s.version = EVC_FIT_STATE_VERSION;
        s.returning = returning ? 1 : 0;
        s.status = returning ? status : 0;
        s.k = k;
        s.evaluations = c.evals;
        s.m = p->m;
        s.hist = hist;
        s.end = end;
        s.low = low ? 1 : 0;
        s.switched_at = switched_at;
        s.n = n;
        s.fx = fx;
        s.negloglk = nll;
        s.xnorm = xnorm;
        s.gnorm = gnorm;
        for (int j = 0; j < p->m; j++) s.ys[j] = sc[2 + j];
        s.yy = sc[0];
        s.seconds = t_offset + elapsed(t_begin);
        const int rc = ckpt(ckpt_user, &s, stream);
        t_saved = std::chrono::steady_clock::now();
        if (rc) { set_error("evc_plm_fit_checkpointed: checkpoint callback failed"); return 1; }
        return 0;
    };
    auto finish_saved = [&](int stat) {
        if (save(true, stat)) return 1;
        return finish(stat);
    };
    // leave the bf16x1 mode: hi+lo products from here on, objective re-evaluated at x[cur], history dropped
    // (a stored pair would mix gradients of two precisions), restart from steepest descent
    auto switch_to_high = [&](int at) -> int {
        if (evc_plm_set_precision(h, 0)) return 1;
        low = false;
        switched_at = at;
        if (fit_evaluate(c, cur, nullptr)) return 1;
        fx = w->h_sc[SC_FX];
        nll = w->h_sc[SC_NLL];
        xnorm = std::sqrt(w->h_sc[SC_XXH] + w->h_sc[SC_XXJ]);
        gnorm = std::sqrt(w->h_sc[SC_GG]);
        hist = 0;
        end = 0;
        pair_pending = false;
        if (fit_direction(c, cur, 0, 0)) return 1;
        step = 1.0 / gnorm;
        return 0;
    };
    if (resume) {
        // the state right after iteration k's progress callback, pair k already stored
        k = resume->k;
        c.evals = resume->evaluations;
        hist = resume->hist;
        end = resume->end;
        low = resume->low != 0;
        switched_at = resume->switched_at;
        fx = resume->fx;
        nll = resume->negloglk;
        xnorm = resume->xnorm;
        gnorm = resume->gnorm;
        if (p->precision_schedule == 1 && evc_plm_set_precision(h, low ? 1 : 0)) return 1;
        double sc[2 + 32];
        sc[0] = resume->yy;
        sc[1] = 0.0;
        for (int j = 0; j < p->m; j++) sc[2 + j] = resume->ys[j];
        EVC_CUDA(cudaMemcpyAsync(w->sc + SC_YY, sc, (2 + p->m) * sizeof(double), cudaMemcpyHostToDevice, st));
        EVC_CUDA(cudaStreamSynchronize(st));
    } else {
        cur = 0;
        if (p->precision_schedule == 1) {
            if (evc_plm_set_precision(h, 1)) return 1;
            low = true;
        }
        EVC_CUDA(cudaMemcpyAsync(w->x[cur], d_x, nb, cudaMemcpyDeviceToDevice, st));
        if (fit_evaluate(c, cur, nullptr)) return 1;
        fx = w->h_sc[SC_FX];
        nll = w->h_sc[SC_NLL];
        xnorm = std::sqrt(w->h_sc[SC_XXH] + w->h_sc[SC_XXJ]);
        gnorm = std::sqrt(w->h_sc[SC_GG]);
        if (gnorm / std::max(1.0, xnorm) <= p->epsilon) {
            if (!low) return finish(EVC_LBFGS_ALREADY_MINIMIZED);
            if (switch_to_high(0)) return 1;
            if (gnorm / std::max(1.0, xnorm) <= p->epsilon) return finish(EVC_LBFGS_ALREADY_MINIMIZED);
        }
        if (fit_direction(c, cur, 0, 0)) return 1;
        step = 1.0 / gnorm;
        k = 1;
    }
    bool resuming = resume != nullptr;
    for (;;) {
        if (!resuming) {
            // ---- line search along d from x[cur] ----
            if (vec_dot(w->g[cur], w->d, n, w->sc + SC_DG, w->partial, st)) return 1;
            EVC_CUDA(cudaMemcpyAsync(w->h_sc, w->sc, 8 * sizeof(double), cudaMemcpyDeviceToHost, st));
            EVC_CUDA(cudaStreamSynchronize(st));
            const double finit = fx, dginit = w->h_sc[SC_DG];
            const int trial = cur ^ 1;
            int ls_status = 0;      // 0 = the line search converged (strong Wolfe conditions hold at `step`)
            int count = 0;
            double f = finit;
            if (step <= 0.0) ls_status = EVC_LBFGSERR_INVALIDPARAMETERS;
            else if (dginit > 0.0) ls_status = EVC_LBFGSERR_INCREASEGRADIENT;
            else {
                MtState ms{0.0, finit, dginit, 0.0, finit, dginit, false};
                bool stage1 = true, uinfo = false;
                const double dgtest = p->ftol * dginit;
                double width = p->max_step - p->min_step, prev_width = 2.0 * width;
                for (;;) {
                    double stmin, stmax;
                    if (ms.brackt) { stmin = std::min(ms.x, ms.y); stmax = std::max(ms.x, ms.y); }
                    else { stmin = ms.x; stmax = step + 4.0 * (step - ms.x); }
                    step = std::min(p->max_step, std::max(p->min_step, step));
                    if ((ms.brackt && ((step <= stmin || stmax <= step) || p->max_linesearch <= count + 1 || uinfo)) ||
                        (ms.brackt && (stmax - stmin <= p->xtol * stmax)))
                        step = ms.x;
                    if (vec_step(w->x[trial], w->x[cur], w->d, (float)step, n, st)) return 1;
                    if (fit_evaluate(c, trial, w->d)) return 1;
                    f = w->h_sc[SC_FX];
                    const double dg = w->h_sc[SC_DG];
                    const double ftest1 = finit + step * dgtest;
                    count++;
                    if (ms.brackt && ((step <= stmin || stmax <= step) || uinfo)) { ls_status = EVC_LBFGSERR_ROUNDING_ERROR; break; }
                    if (step == p->max_step && f <= ftest1 && dg <= dgtest) { ls_status = EVC_LBFGSERR_MAXIMUMSTEP; break; }
                    if (step == p->min_step && (ftest1 < f || dgtest <= dg)) { ls_status = EVC_LBFGSERR_MINIMUMSTEP; break; }
                    if (ms.brackt && (stmax - stmin) <= p->xtol * stmax) { ls_status = EVC_LBFGSERR_WIDTHTOOSMALL; break; }
                    if (p->max_linesearch <= count) { ls_status = EVC_LBFGSERR_MAXIMUMLINESEARCH; break; }
                    if (f <= ftest1 && std::fabs(dg) <= p->gtol * (-dginit)) break;     // accept
                    if (stage1 && f <= ftest1 && std::min(p->ftol, p->gtol) * dginit <= dg) stage1 = false;
                    if (stage1 && ftest1 < f && f <= ms.fx) {
                        MtState m2{ms.x, ms.fx - ms.x * dgtest, ms.dx - dgtest, ms.y, ms.fy - ms.y * dgtest, ms.dy - dgtest,
                                   ms.brackt};
                        uinfo = update_trial_interval(m2, step, f - step * dgtest, dg - dgtest, stmin, stmax);
                        ms = MtState{m2.x, m2.fx + m2.x * dgtest, m2.dx + dgtest, m2.y, m2.fy + m2.y * dgtest,
                                     m2.dy + dgtest, m2.brackt};
                    } else {
                        uinfo = update_trial_interval(ms, step, f, dg, stmin, stmax);
                    }
                    if (ms.brackt) {
                        if (0.66 * prev_width <= std::fabs(ms.y - ms.x)) step = ms.x + 0.5 * (ms.y - ms.x);
                        prev_width = width;
                        width = std::fabs(ms.y - ms.x);
                    }
                }
            }
            if (ls_status != 0) {
                if (low) {
                    // the bf16x1 gradient is no longer good enough for the line search: finish in the hi+lo mode
                    if (switch_to_high(k)) return 1;
                    continue;
                }
                k = k - 1;
                return finish_saved(ls_status);     // x[cur], g[cur] are the last accepted point
            }
            // ---- accepted: x[trial] is the new iterate ----
            cur = trial;
            fx = f;
            nll = w->h_sc[SC_NLL];
            xnorm = std::sqrt(w->h_sc[SC_XXH] + w->h_sc[SC_XXJ]);
            gnorm = std::sqrt(w->h_sc[SC_GG]);
            pair_pending = true;
            if (progress && progress(progress_user, k, fx, xnorm, gnorm, step, count, nll, std::sqrt(w->h_sc[SC_XXH]),
                                     std::sqrt(w->h_sc[SC_XXJ])))
                return finish_saved(EVC_LBFGSERR_CANCELED);
            if (ckpt && ckpt_interval >= 0.0 && elapsed(t_saved) >= ckpt_interval && save(false, 0)) return 1;
        }
        // ---- the iteration boundary: a resumed fit enters here ----
        resuming = false;
        if (low && gnorm / std::max(1.0, xnorm) <= (double)p->switch_factor * p->epsilon) {
            if (switch_to_high(k)) return 1;
            if (gnorm / std::max(1.0, xnorm) <= p->epsilon) return finish_saved(EVC_LBFGS_SUCCESS);
            if (p->max_iterations != 0 && p->max_iterations < k + 1) return finish_saved(EVC_LBFGSERR_MAXIMUMITERATION);
            k++;
            continue;
        }
        if (gnorm / std::max(1.0, xnorm) <= p->epsilon) return finish_saved(EVC_LBFGS_SUCCESS);
        if (p->max_iterations != 0 && p->max_iterations < k + 1) return finish_saved(EVC_LBFGSERR_MAXIMUMITERATION);
        if (pair_pending && add_pair()) return 1;
        k++;
        if (fit_direction(c, cur, hist, end)) return 1;
        // 1 after a pair update; a state without pairs (taken right after the precision switch, or before the first
        // accepted step) continues like the loop does there, from steepest descent with step 1/|g|
        step = hist > 0 ? 1.0 : 1.0 / gnorm;
    }
}

}  // namespace evc

using namespace evc;

extern "C" {

void evc_fit_default_params(evc_fit_params_t *p)
{
    if (!p) return;
    p->max_iterations = 0;
    p->m = 6;
    p->epsilon = 1e-3f;
    p->lambda_h = 0.01f;
    p->lambda_J = 100.f;
    p->max_linesearch = 40;
    p->min_step = 1e-20;
    p->max_step = 1e20;
    p->ftol = 1e-4;
    p->gtol = 0.9;
    p->xtol = 1e-7;
    p->precision_schedule = 0;
    p->switch_factor = 10.f;
}

int evc_plm_fit(evc_plm_t *h, float *d_x, const evc_fit_params_t *p, evc_allreduce_cb allreduce, void *allreduce_user,
                evc_progress_cb progress, void *progress_user, evc_fit_result_t *res, void *stream)
{
    return fit_run(h, d_x, p, allreduce, allreduce_user, progress, progress_user, nullptr, nullptr, -1.0, nullptr, res,
                   stream);
}

int evc_plm_fit_checkpointed(evc_plm_t *h, float *d_x, const evc_fit_params_t *params, evc_allreduce_cb allreduce,
                             void *allreduce_user, evc_progress_cb progress, void *progress_user,
                             evc_checkpoint_cb checkpoint, void *checkpoint_user, double checkpoint_interval,
                             const evc_fit_state_t *resume, evc_fit_result_t *result, void *stream)
{
    return fit_run(h, d_x, params, allreduce, allreduce_user, progress, progress_user, checkpoint, checkpoint_user,
                   checkpoint_interval, resume, result, stream);
}

int evc_plm_fit_prepare(evc_plm_t *h, int32_t m)
{
    if (!h) { set_error("evc_plm_fit_prepare: null handle"); return 1; }
    if (m < 1 || m > 32) { set_error("evc_plm_fit_prepare: history m must be in 1..32"); return 1; }
    if (h->host_pairs > m) {
        set_error("evc_plm_fit_prepare: " + std::to_string(h->host_pairs) + " host-resident correction pairs exceed "
                  "the history m = " + std::to_string(m));
        return 1;
    }
    EVC_CUDA(cudaSetDevice(h->device));
    if (h->fit && (h->fit->m != m || h->fit->host_pairs != h->host_pairs)) {
        fit_work_free(h->fit);
        h->fit = nullptr;
    }
    if (!h->fit) h->fit = fit_work_create(evc_plm_num_params(h), m, h->host_pairs);
    if (!h->fit) return 1;
    h->fit->cur = 0;
    return 0;
}

int evc_plm_fit_vector(evc_plm_t *h, int32_t which, int32_t slot, float **ptr_out)
{
    if (!h || !ptr_out) { set_error("evc_plm_fit_vector: null pointer"); return 1; }
    const FitWork *w = h->fit;
    if (!w) { set_error("evc_plm_fit_vector: no fit workspace (evc_plm_fit_prepare)"); return 1; }
    if (which == EVC_FIT_VEC_X || which == EVC_FIT_VEC_G) {
        *ptr_out = which == EVC_FIT_VEC_X ? w->x[w->cur] : w->g[w->cur];
        return 0;
    }
    if ((which != EVC_FIT_VEC_S && which != EVC_FIT_VEC_Y) || slot < 0 || slot >= w->m) {
        set_error("evc_plm_fit_vector: which must be EVC_FIT_VEC_X, _G, _S or _Y, slot in 0..m-1");
        return 1;
    }
    *ptr_out = which == EVC_FIT_VEC_S ? w->s[slot] : w->y[slot];
    return 0;
}

}  // extern "C"
