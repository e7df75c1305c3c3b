"""
Deterministic synthetic alignments of the BASELINE shapes (SURVEY.md 8d): K = ceil(N/50) random
family centres over the 20 residues, each sequence a copy of a random centre with per-sequence
mutation probability p ~ U(0.1, 0.6) and per-site gap probability 0.05; row 0 (the focus) is gap-free.
Codes are in gap-as-state convention (0 = gap, 1..20 = ACDEFGHIKLMNPQRSTVWY).

``planted_potts_model`` is a Potts model with a few known strong couplings, to be sampled (model_ops.PottsSampler)
into alignments whose contacts are known; ``chain_potts_model`` is a nearest-neighbour chain whose log partition
function is exact by transfer matrices.
"""
import numpy as np

ALPHABET = "-ACDEFGHIKLMNPQRSTVWY"

CONFIG_SEEDS = {1: (200, 40, 1), 2: (50000, 200, 2), 3: (200000, 300, 3), 4: (500000, 500, 4),
                5: (100000, 800, 5)}


def synthetic_msa_codes(N, L, seed, q_res=20, gap_prob=0.05):
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
    return np.where(gaps, 0, codes).astype(np.uint8)


def to_ignore_gaps_codes(codes, q=20):
    """gap-as-state codes (gap 0, residues 1..20) -> ignore_gaps codes (residues 0..19, gap 20)."""
    return np.where(codes == 0, q, codes - 1).astype(np.uint8)


def write_a2m(path, codes, focus_name="seq0", alphabet=ALPHABET):
    """Writes the (N, L) codes as A2M, code k printed as alphabet[k]."""
    N, L = codes.shape
    lut = np.frombuffer(alphabet.encode("ascii"), dtype=np.uint8)
    chars = lut[codes]
    with open(path, "w") as f:
        for n in range(N):
            name = "%s/1-%d" % (focus_name, L) if n == 0 else "seq%d/1-%d" % (n, L)
            f.write(">%s\n%s\n" % (name, bytes(chars[n]).decode("ascii")))


def planted_potts_model(L, q, n_contacts, seed, strength=2.0, field_scale=0.5, alphabet=None):
    """A ``model_ops.read_model``-shaped dict (writable with ``model_io.write_model_file``) with known contacts.

    ``n_contacts`` disjoint site pairs (i, j), |i - j| >= 2, carry a strong block J_ij(a, b) = strength when
    b = pi_ij(a) for a random permutation pi_ij, else 0; every other J is 0, and the fields h_i(a) ~ N(0, field_scale)
    are rounded to multiples of 2^-10.  Deterministic from ``seed``.  ``alphabet`` defaults to the first q characters
    of the protein alphabet with the gap first.  The pairs (0-based sites, i < j) are under "contacts"; f_i and f_ij
    are uniform, and the model holds no sequence weights."""
    alphabet = ALPHABET[:q] if alphabet is None else alphabet
    if len(alphabet) != q:
        raise ValueError("alphabet must have q = %d characters" % q)
    if 2 * n_contacts > L:
        raise ValueError("%d disjoint pairs need at least %d sites" % (n_contacts, 2 * n_contacts))
    rng = np.random.default_rng(seed)
    contacts = []
    for _ in range(1000 * max(1, n_contacts)):
        if len(contacts) == n_contacts:
            break
        i, j = sorted(int(v) for v in rng.choice(L, 2, replace=False))
        used = {k for p in contacts for k in p}
        if j - i >= 2 and i not in used and j not in used:
            contacts.append((i, j))
    if len(contacts) < n_contacts:
        raise ValueError("could not place %d disjoint pairs with |i - j| >= 2 on %d sites" % (n_contacts, L))
    contacts.sort()
    npairs = L * (L - 1) // 2
    J = np.zeros((npairs, q, q), dtype=np.float32)
    for i, j in contacts:
        J[i * L - i * (i + 1) // 2 + (j - i - 1), np.arange(q), rng.permutation(q)] = strength
    h = (np.round(rng.normal(0.0, field_scale, (L, q)) * 1024.0) / 1024.0).astype(np.float32)
    return dict(L=L, q=q, n_valid=0, n_invalid=0, num_iter=0, theta=0.0, lambda_h=0.0, lambda_J=0.0,
                lambda_group=0.0, n_eff=0.0, alphabet=alphabet, weights=np.zeros(0, dtype=np.float32),
                target_seq="".join(alphabet[a] for a in h.argmax(axis=1)), index_list=np.arange(1, L + 1, dtype=np.int32),
                fi=np.full((L, q), 1.0 / q, dtype=np.float32), h=h,
                fij=np.full((npairs, q, q), 1.0 / (q * q), dtype=np.float32), J=J,
                contacts=np.array(contacts, dtype=np.int64).reshape(-1, 2))


def chain_potts_model(L, q, seed, coupling_scale=0.25, field_scale=0.5, alphabet=None):
    """A ``model_ops.read_model``-shaped dict of a nearest-neighbour chain: J_ij is nonzero only for j = i + 1, with
    J_{i,i+1}(a, b) ~ N(0, coupling_scale) and h_i(a) ~ N(0, field_scale), all rounded to multiples of 2^-10 (so the
    sampler's fields are exact in fp32).  Its log partition function is exact by transfer matrices at any L.
    Deterministic from ``seed``; header, f_i and f_ij as in planted_potts_model."""
    alphabet = ALPHABET[:q] if alphabet is None else alphabet
    if len(alphabet) != q:
        raise ValueError("alphabet must have q = %d characters" % q)
    rng = np.random.default_rng(seed)
    npairs = L * (L - 1) // 2
    J = np.zeros((npairs, q, q), dtype=np.float32)
    near = np.array([i * L - i * (i + 1) // 2 for i in range(L - 1)], dtype=np.int64)
    J[near] = np.round(rng.normal(0.0, coupling_scale, (L - 1, q, q)) * 1024.0) / 1024.0
    h = (np.round(rng.normal(0.0, field_scale, (L, q)) * 1024.0) / 1024.0).astype(np.float32)
    return dict(L=L, q=q, n_valid=0, n_invalid=0, num_iter=0, theta=0.0, lambda_h=0.0, lambda_J=0.0,
                lambda_group=0.0, n_eff=0.0, alphabet=alphabet, weights=np.zeros(0, dtype=np.float32),
                target_seq="".join(alphabet[a] for a in h.argmax(axis=1)), index_list=np.arange(1, L + 1, dtype=np.int32),
                fi=np.full((L, q), 1.0 / q, dtype=np.float32), h=h,
                fij=np.full((npairs, q, q), 1.0 / (q * q), dtype=np.float32), J=J)
