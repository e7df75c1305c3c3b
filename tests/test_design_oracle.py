"""CPU checks of design: the float64 restatement on enumerated models (oracle/design.py), the fp32 replay of the
record and the descent with its planted mistakes (oracle/design_replay.py), and the refusals of design_codes and
evcplm-design before any device work."""
import io

import numpy as np
import pytest

from oracle import design as dz
from oracle import design_replay as dr
from oracle import potts_sampler as ps


def random_model(L, q, seed, scale=1.0):
    rng = np.random.default_rng(seed)
    h = rng.normal(0, 0.5 * scale, (L, q)).astype(np.float32)
    J = rng.normal(0, 0.4 * scale, (L * (L - 1) // 2, q, q)).astype(np.float32)
    return h, J


@pytest.mark.parametrize("L, q, seed", [(8, 3, 1), (6, 4, 2)])
def test_restatement_descent_is_local_max_and_anneal_finds_global_max(L, q, seed):
    h, J = random_model(L, q, seed)
    Hmax, _ = dz.global_max(h, J)
    start = ps.uniform_start(seed, 64, L, q)
    codes, settled = dz.descend(h, J, start)
    assert settled.all()
    assert dz.is_local_max(h, J, codes, tol=1e-12).all()
    assert (ps.energies(h, J, codes) <= Hmax + 1e-12).all()
    from evcouplings_b200.model_ops import anneal_schedule
    _E, best = dz.anneal_record(h, J, seed, 64, anneal_schedule(0.2, 4.0, 120))
    final, settled = dz.descend(h, J, best)
    assert settled.all() and dz.is_local_max(h, J, final, tol=1e-12).all()
    assert abs(ps.energies(h, J, final).max() - Hmax) <= 1e-12


def test_restatement_conditional_with_masks():
    L, q = 8, 3
    h, J = random_model(L, q, 5)
    free = np.array([1, 2, 4, 5, 7])
    allowed = np.array([0b011, 0b110, 0b101, 0b111, 0b010])
    context = ps.uniform_start(9, 1, L, q)[0]
    Hmax, argmaxes = dz.global_max(h, J, free, context, allowed)
    start = np.repeat(context[None], 32, axis=0)
    start[:, free] = ps.uniform_start(3, 32, len(free), q)
    codes, settled = dz.descend(h, J, start, free, allowed)
    assert settled.all()
    assert dz.is_local_max(h, J, codes, free, allowed, tol=1e-12).all()
    assert (codes[:, np.setdiff1d(np.arange(L), free)] == context[np.setdiff1d(np.arange(L), free)]).all()
    assert all(((allowed[k] >> codes[:, i]) & 1).all() for k, i in enumerate(free))
    E = ps.energies(h, J, codes)
    assert (E <= Hmax + 1e-12).all()
    assert np.isclose(E.max(), Hmax, rtol=0, atol=1e-12)   # 32 starts over 3 * 2 * 2 * 2 * 3 * 1 states


def generated_calls(kind, mutation=None):
    """A generate-mode trajectory with a record and a descent; returns (replay, constructor of a clean replay)."""
    L, q, C = 10, 4, 8
    h, J = random_model(L, q, 11, scale=1.3)
    if kind == "ties":              # half-integer parameters: exact ties in Z are common
        h, J = np.round(2 * h) / 2, np.round(2 * J) / 2
    if kind == "fresh":             # the descent of design_codes: a new handle, so Z is first built at t = 0
        def make(m=None):
            return dr.DesignReplay(h, J, seed=7, n_chains=C, mutation=m)
        rep = make(mutation)
        rep.descend(40)
    elif kind in ("plain", "ties"):
        def make(m=None):
            return dr.DesignReplay(h, J, seed=7, n_chains=C, mutation=m)
        rep = make(mutation)
        rep.run(3, 1.0)
        rep.record_best()
        rep.run(20, 2.5)
        rep.best()
        rep.run(21, 6.0)            # high beta: chains sit still, so a >= record would move the sweep index
        rep.best()
        rep.descend(13)
        rep.descend(27)             # across the refresh at t = 64
        rep.best()
    elif kind == "tempered":
        def make(m=None):
            return dr.TemperedDesignReplay(h, J, seed=7, n_chains=C, ladder=(0.5, 1.0, 2.0, 8.0), swap_interval=2,
                                           mutation=m)
        rep = make(mutation)
        rep.record_best()
        rep.temper(25)
        rep.best()
        rep.temper(20)
        rep.best()
        rep.descend(40)
    else:
        free = np.array([0, 2, 3, 6, 9])
        allowed = np.array([0b0011, 0b1110, 0b0101, 0b1111, 0b1000])
        from oracle import conditional_sampler as cs
        context = ps.uniform_start(4, C, L, q)
        context[:, 3] = 1           # outside its mask 0b0101: the descent must move it
        hc = cs.fold(h, J, free, context).astype(np.float32)
        Jr = cs.reduced_couplings(J, L, q, free).reshape(len(free), q, len(free), q)
        iu, ju = np.triu_indices(len(free), 1)
        Jred = Jr[iu, :, ju, :].astype(np.float32)

        def make(m=None):
            return dr.DesignReplay(hc[0], Jred, seed=7, n_chains=C, mutation=m, hc=hc, free=free, context=context,
                                   allowed=allowed)
        rep = make(mutation)
        rep.descend(40)
    return rep, make


@pytest.mark.parametrize("kind", ["plain", "ties", "fresh", "tempered", "conditional"])
def test_generated_trajectory_replays_clean(kind):
    rep, make = generated_calls(kind)
    clean = dr.replay_design_calls(make(), rep.calls)
    assert clean.clean(), (clean.violations[:3], clean.descent_violations[:3], clean.record_mismatch[:3])
    assert clean.decisions_checked > 0
    if kind in ("plain", "ties", "tempered"):
        assert clean.n_violations == 0 and clean.checked > 0


@pytest.mark.parametrize("mutation, kind", [("tie_to_smallest", "ties"), ("keep_disallowed", "conditional"),
                                            ("record_ge", "plain"), ("record_before_sweep", "plain"),
                                            ("record_before_sweep", "tempered"),
                                            ("descent_skip_refresh", "fresh")])
def test_planted_mistake_is_caught(mutation, kind):
    bad, make = generated_calls(kind, mutation)
    rep = dr.replay_design_calls(make(), bad.calls)
    assert not rep.clean()


def test_tie_to_smallest_needs_a_tie():
    # an exact tie between the current state and a smaller one: only the rule "keep a tied current state" keeps it
    h = np.zeros((2, 3), dtype=np.float32)
    h[0] = [1.0, 0.0, 1.0]
    J = np.zeros((1, 3, 3), dtype=np.float32)
    good = dr.DesignReplay(h, J, n_chains=1, init=np.array([[2, 0]]))
    bad = dr.DesignReplay(h, J, n_chains=1, init=np.array([[2, 0]]), mutation="tie_to_smallest")
    assert good.descend(1)[0].all() and good.s[0, 0] == 2
    bad.descend(1)
    assert bad.s[0, 0] == 0


def test_python_refusals_before_device_work():
    from evcouplings_b200 import model_ops
    from evcouplings_b200.synthetic import planted_potts_model
    m = planted_potts_model(12, 4, 3, 0)
    for kw in (dict(sweeps=-1), dict(descent_sweeps=-1), dict(beta_start=2.0, beta=1.0), dict(beta=float("nan")),
               dict(beta_start=0.1, ladder=[0.5, 1.0]), dict(ladder=[1.0, 0.5]), dict(free=[10 ** 6]),
               dict(free=[int(m["index_list"][0])], init="random"), dict(num_gpus=0)):
        args = dict(sweeps=4)
        args.update(kw)
        with pytest.raises(ValueError):
            model_ops.design_codes(m, 4, engine=object(), **args)


@pytest.mark.parametrize("argv", [
    ["--sweeps", "-1"], ["--descent-sweeps", "-2"], ["--anneal", "2"], ["--anneal", "0.1", "--ladder", "0.5,1"],
    ["--tempering", "4"], ["--ladder", "1,0.5"], ["--free", "9-3"], ["--allow", "3AV"], ["--gpus", "0"],
    ["--init", "/nonexistent.fasta"], ["--swap-interval", "2"], ["--seed", "-1"]])
def test_command_line_refusals_exit_2(argv, tmp_path):
    from evcouplings_b200 import design_cli
    err = io.StringIO()
    rc = design_cli.main(["model.bin", "-n", "4", "--sweeps", "3", "-o", str(tmp_path / "o.fasta")] + argv,
                         stderr=err)
    assert rc == 2, err.getvalue()
    assert err.getvalue().startswith("evcplm-design:")
    assert not (tmp_path / "o.fasta").exists()


def test_command_line_unknown_position_exits_2(tmp_path):
    from evcouplings_b200 import design_cli
    from evcouplings_b200.synthetic import planted_potts_model
    from test_gpu_conditional_sampler import write_model
    m = planted_potts_model(12, 4, 3, 0)
    path = str(tmp_path / "m.model")
    write_model(path, m)
    err = io.StringIO()
    rc = design_cli.main([path, "-n", "2", "--sweeps", "3", "--init", "target", "--free", "999", "-o",
                          str(tmp_path / "o.fasta")], stderr=err)
    assert rc == 2 and "999" in err.getvalue()


def test_fasta_rows_read_back(tmp_path):
    from evcouplings_b200 import design_cli, sample_cli
    m = dict(L=4, alphabet="ACDE")
    res = dict(codes=np.array([[0, 1, 2, 3], [3, 3, 0, 1]], dtype=np.uint8), energy=np.array([1.5, -2.0]),
               settled=np.array([True, False]), found_at=np.array([7, -1]))
    path = str(tmp_path / "d.fasta")
    design_cli.write_designs(path, res, m["alphabet"])
    lines = open(path).read().splitlines()
    assert lines[0] == ">design_0 H=1.500000 settled=1 found_at=7"
    assert lines[2] == ">design_1 H=-2.000000 settled=0 found_at=-1"
    assert np.array_equal(sample_cli.read_init_file(path, m, 2), res["codes"])
