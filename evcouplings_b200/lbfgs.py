"""
Host-side control logic of the L-BFGS driver (SURVEY.md 8a row a8).

plmc minimises the PLM objective with libLBFGS (recalled, not pinned: history
m = 6, More-Thuente line search, stop when |g| / max(1, |x|) < 1e-3 or at the
iteration cap given by ``-m``; reference flag built at
evcouplings/couplings/tools.py:226-228).  Here the n-vector work lives on the
device behind a small "vector space" object; this module only sees scalars:

    space.evaluate(x)            -> fx (float); the gradient lands in space.g
    space.dot(a, b)              -> float          (a, b: opaque vector handles)
    space.copy(dst, src), space.axpby(y, x, a, b)  (y = a*x + b*y)
    space.direction(d, bound, end)                 two-loop recursion, d = -H g
    space.update_pair(slot, xp, gp) -> (ys, yy)    s = x - xp, y = g - gp into slot
    space.x, space.g, space.xp, space.gp, space.d  vector handles

The product implementation is ``engine.CudaPlmProblem`` (all vector work in
libevcplm kernels); tests drive the same logic with a numpy space.
"""
import math
import time
from collections import namedtuple

LBFGS_SUCCESS = "LBFGS_SUCCESS"
LBFGS_ALREADY_MINIMIZED = "LBFGS_ALREADY_MINIMIZED"
LBFGSERR_MAXIMUMITERATION = "LBFGSERR_MAXIMUMITERATION"
LBFGSERR_MAXIMUMLINESEARCH = "LBFGSERR_MAXIMUMLINESEARCH"
LBFGSERR_MINIMUMSTEP = "LBFGSERR_MINIMUMSTEP"
LBFGSERR_MAXIMUMSTEP = "LBFGSERR_MAXIMUMSTEP"
LBFGSERR_ROUNDING_ERROR = "LBFGSERR_ROUNDING_ERROR"
LBFGSERR_WIDTHTOOSMALL = "LBFGSERR_WIDTHTOOSMALL"
LBFGSERR_INCREASEGRADIENT = "LBFGSERR_INCREASEGRADIENT"
LBFGSERR_CANCELED = "LBFGSERR_CANCELED"

LbfgsParams = namedtuple("LbfgsParams", [
    "m", "epsilon", "max_iterations", "max_linesearch", "min_step", "max_step",
    "ftol", "gtol", "xtol"])


def default_params(max_iterations=0, epsilon=1e-3, m=6):
    return LbfgsParams(m=m, epsilon=epsilon, max_iterations=max_iterations, max_linesearch=40,
                       min_step=1e-20, max_step=1e20, ftol=1e-4, gtol=0.9, xtol=1e-7)


LbfgsResult = namedtuple("LbfgsResult", ["status", "iterations", "fx", "evaluations"])


def _cubic_min(u, fu, du, v, fv, dv):
    d = v - u
    theta = (fu - fv) * 3.0 / d + du + dv
    p, q, r = abs(theta), abs(du), abs(dv)
    s = max(p, q, r)
    a = theta / s
    gamma = s * math.sqrt(max(0.0, a * a - (du / s) * (dv / s)))
    if v < u:
        gamma = -gamma
    p = gamma - du + theta
    q = gamma - du + gamma + dv
    r = p / q
    return u + r * d


def _cubic_min2(u, fu, du, v, fv, dv, xmin, xmax):
    d = v - u
    theta = (fu - fv) * 3.0 / d + du + dv
    p, q, r = abs(theta), abs(du), abs(dv)
    s = max(p, q, r)
    a = theta / s
    gamma = s * math.sqrt(max(0.0, a * a - (du / s) * (dv / s)))
    if u < v:
        gamma = -gamma
    p = gamma - dv + theta
    q = gamma - dv + gamma + du
    r = p / q
    if r < 0.0 and gamma != 0.0:
        return v - r * d
    elif a < 0:
        return xmax
    return xmin


def _quad_min(u, fu, du, v, fv):
    a = v - u
    return u + du / ((fu - fv) / a + du) / 2.0 * a


def _quad_min2(u, du, v, dv):
    a = u - v
    return v + dv / (dv - du) * a


def _update_trial_interval(st, t, ft, dt, tmin, tmax):
    """Safeguarded step update of More & Thuente (1994), sec. 4.
    st = dict(x, fx, dx, y, fy, dy, brackt); returns (new_t, error_flag)."""
    x, fx, dx = st["x"], st["fx"], st["dx"]
    y, fy, dy = st["y"], st["fy"], st["dy"]
    brackt = st["brackt"]
    dsign = (dt * (dx / abs(dx)) < 0.0) if dx != 0.0 else (dt < 0.0)
    if brackt:
        if t <= min(x, y) or max(x, y) <= t:
            return t, True          # trial value out of the interval
        if 0.0 <= dx * (t - x):
            return t, True          # function does not decrease from x
        if tmax < tmin:
            return t, True
    if fx < ft:
        # case 1: higher function value -> minimum bracketed
        brackt = True
        bound = True
        mc = _cubic_min(x, fx, dx, t, ft, dt)
        mq = _quad_min(x, fx, dx, t, ft)
        newt = mc if abs(mc - x) < abs(mq - x) else mc + 0.5 * (mq - mc)
    elif dsign:
        # case 2: lower value, derivatives of opposite sign -> bracketed
        brackt = True
        bound = False
        mc = _cubic_min(x, fx, dx, t, ft, dt)
        mq = _quad_min2(x, dx, t, dt)
        newt = mc if abs(mc - t) > abs(mq - t) else mq
    elif abs(dt) < abs(dx):
        # case 3: lower value, same sign, derivative magnitude decreases
        bound = True
        mc = _cubic_min2(x, fx, dx, t, ft, dt, tmin, tmax)
        mq = _quad_min2(x, dx, t, dt)
        if brackt:
            newt = mc if abs(t - mc) < abs(t - mq) else mq
        else:
            newt = mc if abs(t - mc) > abs(t - mq) else mq
    else:
        # case 4: lower value, same sign, derivative magnitude does not decrease
        bound = False
        if brackt:
            newt = _cubic_min(t, ft, dt, y, fy, dy)
        elif x < t:
            newt = tmax
        else:
            newt = tmin
    # update the interval of uncertainty
    if fx < ft:
        y, fy, dy = t, ft, dt
    else:
        if dsign:
            y, fy, dy = x, fx, dx
        x, fx, dx = t, ft, dt
    newt = min(tmax, max(tmin, newt))
    if brackt and bound:
        mq = x + 0.66 * (y - x)
        if x < y:
            if mq < newt:
                newt = mq
        else:
            if newt < mq:
                newt = mq
    st.update(x=x, fx=fx, dx=dx, y=y, fy=fy, dy=dy, brackt=brackt)
    return newt, False


def line_search_morethuente(phi, finit, dginit, step, p):
    """phi(step) -> (f, dg) evaluates the objective at xp + step*d.
    Returns (status or None, step, f, n_evaluations)."""
    if step <= 0.0:
        return "LBFGSERR_INVALIDPARAMETERS", step, finit, 0
    if dginit > 0.0:
        return LBFGSERR_INCREASEGRADIENT, step, finit, 0
    st = dict(x=0.0, fx=finit, dx=dginit, y=0.0, fy=finit, dy=dginit, brackt=False)
    stage1 = True
    dgtest = p.ftol * dginit
    width = p.max_step - p.min_step
    prev_width = 2.0 * width
    count = 0
    uinfo = False
    f = finit
    while True:
        if st["brackt"]:
            stmin, stmax = min(st["x"], st["y"]), max(st["x"], st["y"])
        else:
            stmin, stmax = st["x"], step + 4.0 * (step - st["x"])
        step = min(p.max_step, max(p.min_step, step))
        if (st["brackt"] and ((step <= stmin or stmax <= step) or p.max_linesearch <= count + 1 or uinfo)) \
                or (st["brackt"] and (stmax - stmin <= p.xtol * stmax)):
            step = st["x"]
        f, dg = phi(step)
        ftest1 = finit + step * dgtest
        count += 1
        if st["brackt"] and ((step <= stmin or stmax <= step) or uinfo):
            return LBFGSERR_ROUNDING_ERROR, step, f, count
        if step == p.max_step and f <= ftest1 and dg <= dgtest:
            return LBFGSERR_MAXIMUMSTEP, step, f, count
        if step == p.min_step and (ftest1 < f or dgtest <= dg):
            return LBFGSERR_MINIMUMSTEP, step, f, count
        if st["brackt"] and (stmax - stmin) <= p.xtol * stmax:
            return LBFGSERR_WIDTHTOOSMALL, step, f, count
        if p.max_linesearch <= count:
            return LBFGSERR_MAXIMUMLINESEARCH, step, f, count
        if f <= ftest1 and abs(dg) <= p.gtol * (-dginit):
            return None, step, f, count
        if stage1 and f <= ftest1 and min(p.ftol, p.gtol) * dginit <= dg:
            stage1 = False
        if stage1 and ftest1 < f and f <= st["fx"]:
            fm = f - step * dgtest
            dgm = dg - dgtest
            st2 = dict(x=st["x"], fx=st["fx"] - st["x"] * dgtest, dx=st["dx"] - dgtest,
                       y=st["y"], fy=st["fy"] - st["y"] * dgtest, dy=st["dy"] - dgtest, brackt=st["brackt"])
            step, uinfo = _update_trial_interval(st2, step, fm, dgm, stmin, stmax)
            st.update(x=st2["x"], fx=st2["fx"] + st2["x"] * dgtest, dx=st2["dx"] + dgtest,
                      y=st2["y"], fy=st2["fy"] + st2["y"] * dgtest, dy=st2["dy"] + dgtest, brackt=st2["brackt"])
        else:
            step, uinfo = _update_trial_interval(st, step, f, dg, stmin, stmax)
        if st["brackt"]:
            if 0.66 * prev_width <= abs(st["y"] - st["x"]):
                step = st["x"] + 0.5 * (st["y"] - st["x"])
            prev_width = width
            width = abs(st["y"] - st["x"])


def minimize(space, params, progress=None, checkpoint=None, checkpoint_interval=-1.0, resume=None):
    """L-BFGS main loop.  ``progress(k, fx, xnorm, gnorm, step, ls_evals)`` is called
    once per iteration; returning True cancels.  Returns LbfgsResult.

    Checkpoints follow evc_plm_fit_checkpointed (include/evcplm.h): ``checkpoint(state)`` receives the state dict
    at an iteration boundary -- every ``checkpoint_interval`` seconds (0: every boundary, < 0: never), when
    ``progress`` cancels, and when the fit returns with a consistent state (``state["reason"]`` is None for the
    interval, else the status).  The pair of iteration k is stored before the call, so the state needs no previous
    iterate; the vectors are space.x, space.g and the ``hist`` slots of space.S / space.Y before ``end``.  With
    ``resume`` (such a state, its vectors loaded into the space) the loop continues after that boundary."""
    m = params.m
    t_begin = time.perf_counter()
    t_saved = t_begin
    if resume is None:
        offset = 0.0
        evals = 1
        fx = space.evaluate(space.x)
        nll = getattr(space, "last_negloglk", float("nan"))
        xnorm = math.sqrt(space.dot(space.x, space.x))
        gnorm = math.sqrt(space.dot(space.g, space.g))
        if gnorm / max(1.0, xnorm) <= params.epsilon:
            return LbfgsResult(LBFGS_ALREADY_MINIMIZED, 0, fx, evals)
        space.axpby(space.d, space.g, -1.0, 0.0)
        step = 1.0 / gnorm
        k, end, hist = 1, 0, 0
    else:
        offset = float(resume["seconds"])
        k, end, hist, evals = int(resume["k"]), int(resume["end"]), int(resume["hist"]), int(resume["evaluations"])
        fx, nll, xnorm, gnorm = resume["fx"], resume["negloglk"], resume["xnorm"], resume["gnorm"]
        space.set_history_scalars(resume["ys"], resume["yy"])
    pending = False                     # the pair of the iteration just accepted is owed

    def add_pair():
        nonlocal hist, end, pending
        space.update_pair(end, space.xp, space.gp)
        hist = min(m, hist + 1)
        end = (end + 1) % m
        pending = False

    def save(reason):
        nonlocal t_saved
        if checkpoint is None:
            return
        if pending:
            add_pair()
        ys, yy = space.get_history_scalars()
        checkpoint(dict(reason=reason, k=k, evaluations=evals, m=m, hist=hist, end=end, low=0, switched_at=-1,
                        n=int(space.n), fx=fx, negloglk=nll, xnorm=xnorm, gnorm=gnorm, ys=[float(v) for v in ys],
                        yy=float(yy), seconds=offset + time.perf_counter() - t_begin))
        t_saved = time.perf_counter()

    def done(status):
        save(status)
        return LbfgsResult(status, k, fx, evals)

    resuming = resume is not None
    while True:
        if not resuming:
            space.copy(space.xp, space.x)
            space.copy(space.gp, space.g)
            dginit = space.dot(space.g, space.d)

            def phi(t):
                # x = xp + t * d
                space.copy(space.x, space.xp)
                space.axpby(space.x, space.d, t, 1.0)
                fval = space.evaluate(space.x)
                return fval, space.dot(space.g, space.d)

            status, step, fnew, n_ls = line_search_morethuente(phi, fx, dginit, step, params)
            evals += n_ls
            if status is not None:
                space.copy(space.x, space.xp)
                space.copy(space.g, space.gp)
                k -= 1
                return done(status)
            fx = fnew
            nll = getattr(space, "last_negloglk", float("nan"))
            xnorm = math.sqrt(space.dot(space.x, space.x))
            gnorm = math.sqrt(space.dot(space.g, space.g))
            pending = True
            if progress is not None and progress(k, fx, xnorm, gnorm, step, n_ls):
                return done(LBFGSERR_CANCELED)
            if checkpoint is not None and 0 <= checkpoint_interval <= time.perf_counter() - t_saved:
                save(None)
        resuming = False
        if gnorm / max(1.0, xnorm) <= params.epsilon:
            return done(LBFGS_SUCCESS)
        if params.max_iterations != 0 and params.max_iterations < k + 1:
            return done(LBFGSERR_MAXIMUMITERATION)
        if pending:
            add_pair()
        k += 1
        space.direction(space.d, hist, end)
        step = 1.0 if hist > 0 else 1.0 / gnorm
