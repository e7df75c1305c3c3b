"""
TEST INFRASTRUCTURE -- NOT PRODUCT CODE.

CPU oracle: a plain numpy / float64 restatement of the algorithm that the
EVcouplings pipeline delegates to the external ``plmc`` C/OpenMP binary
(reference call site: evcouplings/couplings/tools.py:202-266, caller
evcouplings/couplings/protocol.py:203-218).  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl
reference`` legs may import this module; the product package
(``evcouplings_b200``) never does.

plmc itself (github.com/debbiemarkslab/plmc, no pinned version --
reference README.md:35-42 only says "compile using make all-openmp32") is NOT
vendored with the reference and cannot be built here.  Parity is therefore
pinned against the *outputs of a real plmc run* that the reference ships in
notebooks/example/ (PABP_YEAST.a2m / .model_params / _ECs.txt) -- see
tests/golden/make_golden.py and tests/test_oracle_golden.py:

  * validity / focus-column rule ........ exact  (151496 valid + 545 invalid, 82 of 96 sites)
  * Hamming neighbour counts ............ exact integers (stored in the golden ``weights``)
  * f_i / f_ij ........................... <= 1e-6 vs golden
  * EC text (APC of Frobenius norms) ..... <= 1e-6 vs golden _ECs.txt from golden J
  * objective scaling .................... data-gradient / (2 lambda_J J) ~ 0.97-0.99 at the golden optimum

What is NOT pinned by any file in the reference (no plmc source, no plmc
tests): the L-BFGS trajectory (initial point, line search, epsilon, history
size).  The objective is strictly convex (lambda > 0) so these change the path
but not the optimum; parity tests therefore compare at convergence.

Parameter vector layout everywhere (identical to the plmc_v2 ``.model`` file,
evcouplings/couplings/model.py:354-389): ``x = [h (L*q) | J (L(L-1)/2 blocks of
q*q, pairs i<j in row-major (i,j) order, block[a][b] with a = state at i)]``.
"""
import numpy as np

GAP = "-"
ALPHABET_PROTEIN = "-ACDEFGHIKLMNPQRSTVWY"   # evcouplings/align/alignment.py:21-26


# --------------------------------------------------------------------------
# a4: MSA ingest, validity filter, focus columns (SURVEY 8a row a4, facts (E))
# --------------------------------------------------------------------------
def read_a2m(path):
    """Minimal FASTA/A2M reader (same record semantics as
    evcouplings/align/alignment.py:42-74 read_fasta)."""
    ids, seqs, cur = [], [], None
    with open(path) as f:
        for line in f:
            line = line.rstrip("\n").rstrip("\r")
            if line.startswith(">"):
                if cur is not None:
                    seqs.append("".join(cur))
                ids.append(line[1:].strip())
                cur = []
            elif cur is not None:
                cur.append(line.strip())
    if cur is not None:
        seqs.append("".join(cur))
    return ids, seqs


def prepare_alignment(ids, seqs, focus=None, alphabet=None, ignore_gaps=False):
    """
    Restates plmc's alignment preparation as pinned by the golden run:

    * every row is upper-cased; '.' is a gap;
    * a row is INVALID if any character anywhere in the row (insert columns
      included) is outside alphabet U {'-', '.'}  (PABP: 545 invalid);
    * in focus mode the model sites are the columns where the focus sequence
      has an upper-case non-gap character (PABP: 96 -> 82);
    * index_list = region_start + residue offset of the focus sequence.

    Returns dict with ``codes`` (N_valid x L uint8), ``valid`` mask over all
    rows, ``q`` (model states), ``gap_code`` (-1 if gap is a model state).
    In gap-as-state mode code == index in ``alphabet`` (gap = 0); with
    ignore_gaps the residues are 0..q-1 in alphabet[1:] order and gap = q.
    """
    if alphabet is None:
        alphabet = ALPHABET_PROTEIN
    gap = alphabet[0]
    n_total = len(seqs)
    width = len(seqs[0])

    focus_index = None
    region_start = 1
    if focus is not None:
        key = focus.split("/")[0]
        for k, name in enumerate(ids):
            tok = name.split()[0] if name.split() else name
            if tok == focus or tok.split("/")[0] == key:
                focus_index = k
                break
        if focus_index is None:
            raise ValueError("focus sequence not found: " + focus)
        name = ids[focus_index].split()[0]
        if "/" in name:
            try:
                region_start = int(name.split("/")[-1].split("-")[0])
            except ValueError:
                region_start = 1
        fseq = seqs[focus_index]
        cols, index_list, offset = [], [], 0
        for c, ch in enumerate(fseq):
            if ch in (gap, "."):
                continue
            if ch == ch.upper():
                cols.append(c)
                index_list.append(region_start + offset)
            offset += 1
    else:
        cols = list(range(width))
        index_list = list(range(1, width + 1))

    allowed = set(alphabet) | {"-", "."}
    lut = {}
    if ignore_gaps:
        q = len(alphabet) - 1
        for k, ch in enumerate(alphabet[1:]):
            lut[ch] = k
        lut[gap] = q
        lut["-"] = q
        lut["."] = q
        gap_code = q
        model_alphabet = alphabet[1:]
    else:
        q = len(alphabet)
        for k, ch in enumerate(alphabet):
            lut[ch] = k
        lut["-"] = 0
        lut["."] = 0
        gap_code = -1
        model_alphabet = alphabet

    valid = np.zeros(n_total, dtype=bool)
    rows = []
    for s, seq in enumerate(seqs):
        up = seq.upper()
        if len(up) != width:
            raise ValueError("ragged alignment at row %d" % s)
        if all(ch in allowed for ch in up):
            valid[s] = True
            rows.append([lut[up[c]] for c in cols])
    codes = np.array(rows, dtype=np.uint8).reshape(len(rows), len(cols))
    target = "".join(seqs[focus_index].upper()[c] for c in cols) if focus_index is not None \
        else "".join(seqs[0].upper()[c].replace(".", "-") for c in cols)
    return dict(
        codes=codes, valid=valid, q=q, gap_code=gap_code,
        model_alphabet=model_alphabet, focus_index=focus_index,
        focus_cols=np.array(cols, dtype=np.int64),
        index_list=np.array(index_list, dtype=np.int32),
        target_seq=target, region_start=region_start,
        n_total=n_total, n_valid=int(valid.sum()),
        num_total_sites=width if focus_index is None else
        sum(1 for ch in seqs[focus_index] if ch not in (gap, ".")),
    )


# --------------------------------------------------------------------------
# a5: Hamming sequence reweighting  (hot path (b))
# --------------------------------------------------------------------------
def identity_threshold_count(theta, L):
    """Smallest integer c with c / float(L) >= theta -- the integer form of
    the in-tree rule ``pair_id / L >= identity_threshold``
    (evcouplings/align/alignment.py:1229)."""
    c = int(np.floor(theta * L))
    while c > 0 and (c - 1) / float(L) >= theta:
        c -= 1
    while c / float(L) < theta:
        c += 1
    return c


def hamming_counts(codes, theta):
    """n_s = #{t : sum_k [code_sk == code_tk] >= theta*L}, self included,
    gap==gap counts as identity (SURVEY row a5 (E); in-tree twin
    evcouplings/align/alignment.py:1192-1233).  ``theta`` in EVcouplings
    convention (identity threshold, e.g. 0.8)."""
    N, L = codes.shape
    thr = identity_threshold_count(theta, L)
    counts = np.zeros(N, dtype=np.int64)
    blk = max(1, int(2e7 // max(1, N * 1)))
    blk = min(max(blk, 16), 512)
    for s0 in range(0, N, blk):
        a = codes[s0:s0 + blk]
        ident = np.zeros((a.shape[0], N), dtype=np.int32)
        for k in range(L):
            ident += (a[:, k:k + 1] == codes[None, :, k])
        counts[s0:s0 + blk] = (ident >= thr).sum(axis=1)
    return counts


def sequence_weights(counts, scale=1.0):
    return scale / counts.astype(np.float64)


# --------------------------------------------------------------------------
# operand rounding of the tensor-core products (plm_tc.cu): a float64 model of
# what the bf16 operands hold, so that the device can be checked against the
# same arithmetic instead of against exact operands
# --------------------------------------------------------------------------
def rn_bf16(v):
    """float32 values rounded to bfloat16 (round to nearest, ties to even), returned as float32: the bit
    operation behind __float2bfloat16_rn.  NaN stays NaN; values that round past the largest bfloat16
    become +-inf."""
    a = np.ascontiguousarray(v, dtype=np.float32)
    u = a.view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    out = u.astype(np.uint32).view(np.float32).reshape(a.shape)
    return np.where(np.isnan(a), a, out)


def bf16_operand(v, operands):
    """The value an operand of the tensor-core GEMMs holds for the float32 value of ``v``, in float64:
    "hi" -> rn_bf16(v) (precision mode 1, bf16 tiles); "hi+lo" -> rn_bf16(v) + rn_bf16(v - rn_bf16(v))
    (precision mode 0; the difference is exact in float32, the pair keeps 16 mantissa bits)."""
    if operands not in ("hi", "hi+lo"):
        raise ValueError("operands must be None, 'hi' or 'hi+lo'")
    v32 = np.asarray(v, dtype=np.float32)
    hi = rn_bf16(v32)
    if operands == "hi":
        return hi.astype(np.float64)
    return hi.astype(np.float64) + rn_bf16(v32 - hi).astype(np.float64)


# --------------------------------------------------------------------------
# a6: single / pair frequencies as written to the .model file
# --------------------------------------------------------------------------
def one_hot(codes, q):
    """N x L x q one-hot; codes >= q (the ignore_gaps gap code) give a zero row."""
    N, L = codes.shape
    X = np.zeros((N, L, q))
    n_idx, l_idx = np.nonzero(codes < q)
    X[n_idx, l_idx, codes[n_idx, l_idx]] = 1.0
    return X


def frequencies(codes, w, q, gap_code=-1, weights=None):
    """f_i (L x q) and f_ij as tri blocks (npairs x q x q).
    gap-as-state: divide by N_eff (alignment.py:1106,1144).
    ignore_gaps:  per-site / per-pair normalisation over non-gap weight
                  (SURVEY row a6 (E), max diff vs golden 5e-10).
    weights="hi+lo": the pair counts take each weight as the tensor-core backward product sees it,
    bf16 hi + lo of its float32 value (16 mantissa bits, see bf16_operand); f_i and N_eff keep the weights
    as given.  None: exact weights everywhere."""
    N, L = codes.shape
    X = one_hot(codes, q)
    Xw = X * w[:, None, None]
    fi = Xw.sum(axis=0)
    if weights is not None:
        Xw = X * bf16_operand(w, weights)[:, None, None]
    F = np.einsum("nia,njb->ijab", Xw, X, optimize=True)
    if gap_code < 0:
        neff = w.sum()
        fi = fi / neff
        F = F / neff
    else:
        fi = fi / np.maximum(fi.sum(axis=1, keepdims=True), 1e-300)
        F = F / np.maximum(F.sum(axis=(2, 3), keepdims=True), 1e-300)
    iu, ju = np.triu_indices(L, 1)
    return fi, F[iu, ju]


# --------------------------------------------------------------------------
# a7: PLM negative log-posterior + gradient  (hot path (a))
# --------------------------------------------------------------------------
def unpack(x, L, q):
    h = x[:L * q].reshape(L, q)
    Jt = x[L * q:].reshape(L * (L - 1) // 2, q, q)
    return h, Jt


def full_couplings(Jt, L, q):
    J = np.zeros((L, L, q, q))
    iu, ju = np.triu_indices(L, 1)
    J[iu, ju] = Jt
    J[ju, iu] = Jt.transpose(0, 2, 1)
    return J


def objective(x, codes, w, q, lambda_h, lambda_J, gap_code=-1, chunk=4096, operands=None, bounds=None):
    """
    F(h,J) = - sum_s w_s sum_i log softmax_a( h_i(a) + sum_{j!=i} J_ij(a, s_j) )[s_i]
             + lambda_h sum h^2 + lambda_J sum_{i<j,a,b} J_ij(a,b)^2
    with un-normalised weights, J shared by the two conditionals, gradient of
    the penalty 2*lambda*x (SURVEY row a7 (E)).  ignore_gaps: site i skipped
    when s_i is a gap; a gapped s_j adds nothing to the logits and gets no
    gradient.  Returns (fx, g, negloglk) in float64.

    operands="hi+lo" / "hi": the arithmetic of the tensor-core path in precision
    mode 0 / 1 (plm_tc.cu), every sum still in float64.  The couplings enter the
    logits as bf16_operand of their float32 value (expand_tc_kernel; the one-hot
    operand is exact); the residuals r = w (p - onehot) of those logits enter the
    pair gradient as bf16_operand(float32(r)) (plm_softmax_kernel); g_h and fx
    use the unrounded residuals and logits.  None: exact operands.

    bounds=nu (with operands): also return a dict of per-entry scales of the
    gradient (in its layout), for error models of a device evaluation: "g_abs"
    (the sum of |terms| of every entry) and "g_flip" (the pair
    gradient's sum of the largest change of a residual operand when the residual
    itself moves by up to nu * w, i.e. operands that can round to a neighbouring
    bf16 value under float32 noise of that size).
    """
    x = np.asarray(x, dtype=np.float64)
    N, L = codes.shape
    h, Jt = unpack(x, L, q)
    J = full_couplings(Jt, L, q)                       # [i, j, a, b]
    W = J.transpose(1, 3, 0, 2).reshape(L * q, L * q)  # [(j,b), (i,a)]
    if bounds is not None and operands is None:
        raise ValueError("bounds= models the rounding of operands= 'hi' or 'hi+lo'")
    if operands is not None:
        W = bf16_operand(W, operands)
    fx = 0.0
    gh = np.zeros((L, q))
    G = np.zeros((L * q, L * q))                       # [(j,b), (i,a)]
    if bounds is not None:
        gh_abs, G_abs, G_flip = np.zeros((L, q)), np.zeros_like(G), np.zeros_like(G)
    for s0 in range(0, N, chunk):
        c = codes[s0:s0 + chunk]
        ww = w[s0:s0 + chunk]
        X = one_hot(c, q)                              # n, L, q
        Xf = X.reshape(len(c), L * q)
        Z = (Xf @ W).reshape(len(c), L, q) + h[None]
        Z -= Z.max(axis=2, keepdims=True)
        lse = np.log(np.exp(Z).sum(axis=2, keepdims=True))
        logP = Z - lse
        P = np.exp(logP)
        present = X.sum(axis=2)                        # 1 unless gap under ignore_gaps
        fx -= (ww[:, None] * (logP * X).sum(axis=2)).sum()
        R = ww[:, None, None] * present[:, :, None] * (P - X)
        gh += R.sum(axis=0)
        R2 = R.reshape(len(c), L * q)
        Rop = R2 if operands is None else bf16_operand(R2, operands)
        G += Xf.T @ Rop
        if bounds is not None:
            gh_abs += np.abs(R).sum(axis=0)
            G_abs += Xf.T @ np.abs(Rop)
            nu = np.repeat(bounds * ww[:, None] * present, q, axis=1)          # [n, (i,a)]
            flip = np.maximum(np.abs(bf16_operand(R2 + nu, operands) - Rop),
                              np.abs(bf16_operand(R2 - nu, operands) - Rop))
            G_flip += Xf.T @ flip
    iu, ju = np.triu_indices(L, 1)

    def pairs(M):
        M4 = M.reshape(L, q, L, q)                      # [j, b, i, a]
        # block (i<j)[a][b] gets conditional i: M4[j,b,i,a] and conditional j: M4[i,a,j,b]
        return M4[ju, :, iu, :].transpose(0, 2, 1) + M4[iu, :, ju, :]
    gJ = pairs(G)
    negloglk = fx
    fx = fx + lambda_h * (h ** 2).sum() + lambda_J * (Jt ** 2).sum()
    g = np.concatenate([(gh + 2 * lambda_h * h).ravel(),
                        (gJ + 2 * lambda_J * Jt).ravel()])
    if bounds is not None:
        return fx, g, negloglk, dict(g_abs=np.concatenate([gh_abs.ravel(), pairs(G_abs).ravel()]),
                                     g_flip=np.concatenate([np.zeros(L * q), pairs(G_flip).ravel()]))
    return fx, g, negloglk


def objective_loops(x, codes, w, q, lambda_h, lambda_J, gap_code=-1):
    """Pure-python-loop statement of the same objective, written directly from
    the formula (tiny cases only); used to check the vectorised version."""
    N, L = codes.shape
    h, Jt = unpack(np.asarray(x, dtype=np.float64), L, q)
    J = full_couplings(Jt, L, q)
    fx = 0.0
    gh = np.zeros_like(h)
    gJf = np.zeros_like(J)
    for s in range(N):
        for i in range(L):
            si = codes[s, i]
            if si >= q:
                continue
            z = h[i].copy()
            for j in range(L):
                sj = codes[s, j]
                if j != i and sj < q:
                    z += J[i, j, :, sj]
            z -= z.max()
            p = np.exp(z) / np.exp(z).sum()
            fx -= w[s] * np.log(p[si])
            r = w[s] * p
            r[si] -= w[s]
            gh[i] += r
            for j in range(L):
                sj = codes[s, j]
                if j != i and sj < q:
                    gJf[i, j, :, sj] += r
    iu, ju = np.triu_indices(L, 1)
    gJ = gJf[iu, ju] + gJf[ju, iu].transpose(0, 2, 1)
    nll = fx
    fx += lambda_h * (h ** 2).sum() + lambda_J * (Jt ** 2).sum()
    g = np.concatenate([(gh + 2 * lambda_h * h).ravel(), (gJ + 2 * lambda_J * Jt).ravel()])
    return fx, g, nll


def initial_point(fi, L, q, n_eff):
    """Independent-site start (plmc behaviour recalled, not pinned (M)):
    h = log of pseudo-counted f_i, centred per site; J = 0."""
    h = np.log((fi * n_eff + 1.0) / (n_eff + q))
    h -= h.mean(axis=1, keepdims=True)
    return np.concatenate([h.ravel(), np.zeros(L * (L - 1) // 2 * q * q)])


def fit(codes, w, q, lambda_h, lambda_J, gap_code=-1, x0=None, max_iter=2000,
        gtol=1e-9, objective_fn=None):
    """Minimise the (strictly convex) objective in float64 with scipy's
    L-BFGS-B -- an implementation independent of the product's L-BFGS."""
    from scipy.optimize import minimize
    N, L = codes.shape
    n = L * q + L * (L - 1) // 2 * q * q
    if x0 is None:
        x0 = np.zeros(n)

    def fun(x):
        if objective_fn is not None:       # e.g. the C/OpenMP float64 port (same objective, faster)
            fx, g, _ = objective_fn(x)
        else:
            fx, g, _ = objective(x, codes, w, q, lambda_h, lambda_J, gap_code)
        return fx, g

    res = minimize(fun, x0, jac=True, method="L-BFGS-B",
                   options=dict(maxiter=max_iter, maxfun=4 * max_iter, maxcor=20,
                                ftol=1e-15, gtol=gtol))
    return res.x, res


# --------------------------------------------------------------------------
# a10: EC scores as plmc writes them (raw gauge Frobenius norm + APC)
# --------------------------------------------------------------------------
def fn_scores(Jt, L):
    F = np.zeros((L, L))
    iu, ju = np.triu_indices(L, 1)
    F[iu, ju] = np.sqrt((Jt.astype(np.float64) ** 2).sum(axis=(1, 2)))
    return F + F.T


def cn_scores(Jt, L):
    """cn_ij = F_ij - c_i c_j / cbar, F = Frobenius norm of J_ij in the gauge
    of the file (no zero-sum shift): SURVEY row a10 (E), rms 2.9e-7 vs golden."""
    F = fn_scores(Jt, L)
    ci = F.sum(axis=1) / (L - 1)
    cbar = F.sum() / (L * (L - 1))
    C = F - np.outer(ci, ci) / cbar
    iu, ju = np.triu_indices(L, 1)
    return C[iu, ju]


def write_ecs(path, Jt, L, index_list, target_seq):
    """Text format read by evcouplings/couplings/pairs.py:55-58."""
    cn = cn_scores(Jt, L)
    iu, ju = np.triu_indices(L, 1)
    with open(path, "w") as f:
        for k in range(len(iu)):
            i, j = iu[k], ju[k]
            f.write("%d %s %d %s 0 %f\n" % (index_list[i], target_seq[i],
                                            index_list[j], target_seq[j], cn[k]))


# --------------------------------------------------------------------------
# a9: plmc_v2 .model writer (layout: evcouplings/couplings/model.py:317-389)
# --------------------------------------------------------------------------
def write_model(path, L, q, n_valid, n_invalid, num_iter, theta_plmc, lambda_h,
                lambda_J, lambda_group, n_eff, alphabet, weights_all, target_seq,
                index_list, fi, h, fij_tri, J_tri):
    with open(path, "wb") as f:
        np.array([L, q, n_valid, n_invalid, num_iter], dtype="<i4").tofile(f)
        np.array([theta_plmc, lambda_h, lambda_J, lambda_group, n_eff], dtype="<f4").tofile(f)
        f.write(alphabet.encode("ascii"))
        np.asarray(weights_all, dtype="<f4").tofile(f)
        f.write(target_seq.encode("ascii"))
        np.asarray(index_list, dtype="<i4").tofile(f)
        np.asarray(fi, dtype="<f4").tofile(f)
        np.asarray(h, dtype="<f4").tofile(f)
        np.asarray(fij_tri, dtype="<f4").tofile(f)
        np.asarray(J_tri, dtype="<f4").tofile(f)


def read_model(path):
    """Bulk reader of the plmc_v2 layout (same byte order as
    evcouplings/couplings/model.py:317-389, tri blocks kept packed)."""
    with open(path, "rb") as f:
        L, q, nv, ni, it = np.fromfile(f, "<i4", 5)
        theta, lh, lj, lg, neff = np.fromfile(f, "<f4", 5)
        alphabet = f.read(q).decode("ascii")
        weights = np.fromfile(f, "<f4", nv + ni)
        target = f.read(L).decode("ascii")
        index_list = np.fromfile(f, "<i4", L)
        fi = np.fromfile(f, "<f4", L * q).reshape(L, q)
        h = np.fromfile(f, "<f4", L * q).reshape(L, q)
        npair = L * (L - 1) // 2
        fij = np.fromfile(f, "<f4", npair * q * q).reshape(npair, q, q)
        J = np.fromfile(f, "<f4", npair * q * q).reshape(npair, q, q)
        rest = f.read()
    assert len(rest) == 0, "trailing bytes in model file"
    return dict(L=int(L), q=int(q), n_valid=int(nv), n_invalid=int(ni), num_iter=int(it),
                theta=float(theta), lambda_h=float(lh), lambda_J=float(lj),
                lambda_group=float(lg), n_eff=float(neff), alphabet=alphabet,
                weights=weights, target_seq=target, index_list=index_list,
                fi=fi, h=h, fij=fij, J=J)


# --------------------------------------------------------------------------
# synthetic MSA generator (SURVEY 8d)
# --------------------------------------------------------------------------
def synthetic_msa_codes(N, L, seed, q_res=20, gap_prob=0.05):
    """Deterministic family-structured synthetic alignment, gap-as-state codes
    (0 = gap, 1..20 residues); row 0 (the focus) is gap-free.  Mirrors
    evcouplings_b200.synthetic.synthetic_msa_codes (kept separate on purpose)."""
    rng = np.random.default_rng(seed)
    K = max(1, -(-N // 50))
    centres = rng.integers(1, q_res + 1, size=(K, L), dtype=np.uint8)
    which = rng.integers(0, K, size=N)
    p_mut = rng.uniform(0.1, 0.6, size=N)
    codes = centres[which]
    mut = rng.random((N, L)) < p_mut[:, None]
    rnd = rng.integers(1, q_res + 1, size=(N, L), dtype=np.uint8)
    codes = np.where(mut, rnd, codes)
    gaps = rng.random((N, L)) < gap_prob
    gaps[0, :] = False
    codes = np.where(gaps, 0, codes).astype(np.uint8)
    return codes
