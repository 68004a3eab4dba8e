"""CPU: the ``grid_dtype`` option of the four GP choosers -- parsing, validation, hand-over to the lazily made
DeviceBackend -- and that ``grid_dtype=float64`` leaves the host logic alone: on the oracle backend every chooser
reproduces its golden next() run (proposal, chain) and leaves the same pickle and global RNG state as the default."""
import pickle

import numpy as np
import pytest

from tests.helpers import hypers, load

CHOOSERS = ("GPEIChooserB200", "GPEIOptChooserB200", "GPEIperSecChooserB200", "GPConstrainedEIChooserB200")


def _mod(name):
    import importlib
    return importlib.import_module("spearmint_b200.chooser." + name)


@pytest.mark.parametrize("name", CHOOSERS)
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_arg_string_accepts_grid_dtype(name, dtype, tmp_path):
    ch = _mod(name).init(str(tmp_path), "mcmc_iters=2,grid_dtype=%s" % dtype)
    assert ch._grid_dtype == dtype
    assert ch._backend is None                               # nothing made on the device yet


@pytest.mark.parametrize("name", CHOOSERS)
@pytest.mark.parametrize("bad", ["float16", "double", "", "Float64"])
def test_bad_grid_dtype_raises_value_error(name, bad, tmp_path):
    with pytest.raises(ValueError):
        _mod(name).init(str(tmp_path), "grid_dtype=%s" % bad)


def test_default_is_float32(tmp_path):
    for name in CHOOSERS:
        assert _mod(name).init(str(tmp_path), "")._grid_dtype == "float32"


def test_random_forest_chooser_rejects_the_option(tmp_path):
    """Unknown keys give TypeError there, as in the reference; the forest has no grid-pass precision to choose."""
    with pytest.raises(TypeError):
        _mod("RandomForestEIChooserB200").init(str(tmp_path), "grid_dtype=float64")


@pytest.mark.parametrize("name", CHOOSERS)
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_lazy_backend_receives_grid_dtype(name, dtype, tmp_path, monkeypatch):
    from spearmint_b200 import backend as B
    made = []

    class Fake(object):
        def __init__(self, device=None, refine_dtype="float64", grid_dtype="float32"):
            made.append(dict(device=device, refine_dtype=refine_dtype, grid_dtype=grid_dtype))

    monkeypatch.setattr(B, "DeviceBackend", Fake)
    ch = _mod(name).init(str(tmp_path), "grid_dtype=%s,device=cuda:3" % dtype)
    assert isinstance(ch.backend, Fake) and ch.backend is ch.backend
    assert made == [dict(device="cuda:3", refine_dtype="float64", grid_dtype=dtype)]


def test_device_backend_validates_grid_dtype():
    """Checked before any engine (or CUDA context) is made."""
    from spearmint_b200.backend import DeviceBackend
    with pytest.raises(ValueError):
        DeviceBackend(grid_dtype="float16")


# ------------------------------------------------------------------------------------------- golden next() runs
def _rng():
    st = np.random.get_state()
    return np.r_[st[1], st[2]]


def _state_bytes(ch):
    with open(ch.state_pkl, "rb") as fh:
        raw = fh.read()
    assert pickle.loads(raw)                                 # a readable state pickle
    return raw


def _run(mod_name, args, g, backend, tmp_path):
    ch = _mod(mod_name).init(str(tmp_path), args)
    ch._backend = backend
    np.random.seed(int(g["seed"]))
    ret = ch.next(g["grid"], g["values"], g["durations"], g["candidates"], g["pending"], g["complete"])
    if hasattr(ch, "dump_hypers") and mod_name == "GPEIChooserB200":
        ch.dump_hypers()
    return ch, ret, _rng()


def _check_ret(ret, g):
    if int(g.get("next_is_tuple", 0)):
        assert isinstance(ret, tuple) and ret[0] == int(g["next_index"])
        np.testing.assert_allclose(ret[1], g["next_point"], rtol=0, atol=1e-6)
    else:
        assert isinstance(ret, int) and ret == int(g["next_index"])


@pytest.mark.parametrize("mod_name,case,args", [
    ("GPEIOptChooserB200", "opt_d8_m52_pend",
     "covar={kind},mcmc_iters={S},burnin={burnin},noiseless={noiseless},use_multiprocessing=0,grid_subset=5"),
    ("GPEIOptChooserB200", "opt_branin2d",
     "covar={kind},mcmc_iters={S},burnin={burnin},noiseless={noiseless},use_multiprocessing=0,grid_subset=5"),
    ("GPEIperSecChooserB200", "psec_d3_pend", "covar={kind},mcmc_iters={S},burnin={burnin},grid_subset=4"),
    ("GPEIChooserB200", "gpei_d3", "mcmc_iters=4"),
])
def test_float64_grid_reproduces_golden_next(mod_name, case, args, tmp_path):
    from tests.oracle_backend import OracleBackend
    g = load(case)
    a = args.format(kind=str(g["kind"]) if "kind" in g else "", S=int(g["S"]) if "S" in g else 0,
                    burnin=int(g["burnin"]) if "burnin" in g else 0,
                    noiseless=int(g["noiseless"]) if "noiseless" in g else 0)
    (tmp_path / "a").mkdir()
    (tmp_path / "b").mkdir()
    ch0, ret0, rng0 = _run(mod_name, a, g, OracleBackend(), tmp_path / "a")
    ch1, ret1, rng1 = _run(mod_name, a + ",grid_dtype=float64", g, OracleBackend(), tmp_path / "b")
    assert ch1._grid_dtype == "float64"
    _check_ret(ret1, g)
    assert ret1 == ret0 if not isinstance(ret0, tuple) else (ret1[0] == ret0[0] and np.array_equal(ret1[1], ret0[1]))
    if mod_name != "GPEIChooserB200":
        for a_, b_ in zip(ch1.hyper_samples, hypers(g)):
            np.testing.assert_allclose(np.hstack(a_), np.hstack(b_), rtol=1e-9)
        assert [np.hstack(h).tolist() for h in ch1.hyper_samples] == [np.hstack(h).tolist() for h in ch0.hyper_samples]
    np.testing.assert_array_equal(rng1, rng0)
    assert _state_bytes(ch1) == _state_bytes(ch0)            # byte for byte
    if hasattr(ch1, "stats_file") and mod_name == "GPEIOptChooserB200":
        assert open(ch1.stats_file).read() == open(ch0.stats_file).read()


@pytest.mark.parametrize("case", ["cons_next_vanilla.npz", "cons_next_nan_pend_d3.npz"])
def test_float64_grid_reproduces_golden_next_constrained(case, tmp_path, monkeypatch):
    from spearmint_b200.chooser import GPConstrainedEIChooserB200 as CB
    from tests.constrained_oracle_backend import ConstrainedOracleBackend
    from tests.test_constrained_chooser import GOLDEN_NEXT, check_against_golden, run_plugin
    path = [p for p in GOLDEN_NEXT if p.endswith(case)][0]
    init = CB.init
    made = []

    def init64(expt_dir, opts):
        ch = init(expt_dir, opts + ",grid_dtype=float64")
        made.append(ch)
        return ch
    monkeypatch.setattr(CB, "init", init64)
    z, out, ncalls = run_plugin(path, ConstrainedOracleBackend(), tmp_path)
    assert made and made[0]._grid_dtype == "float64"
    check_against_golden(z, out, ncalls, rtol=1e-8, atol_point=1e-6)
