"""smk_predict_mma_f64 (csrc/predict_mma.cu): the float64 fused predict on the fp64 tensor cores, against the SIMT float64
kernel smk_predict_f64 on the same device factor, and against the float64 oracle (scipy Cholesky + solve_triangular).

The two kernels evaluate the same expressions from the same L, winv and alpha; only the summation order of the
substitution and of the column reductions differs.  So mu and var must agree to 1e-11 of amp2, at every block count
(N = 1 ... 8192: 1 to 64 row blocks of 64), candidate tile count (M = 1 ... 10 010: ragged last tiles of 64), sample
count (S = 1 ... 40: the sample-major work list) and dimension (D = 1, 8, 32: one or several generator chunks), for all
four kernels.  Against the oracle the kernel must be as close as the SIMT kernel is, up to the same 1e-11 amp2.
"""
import numpy as np
import pytest

from tests.helpers import cur_stream, data, lib, synth_hypers

gpu = pytest.mark.gpu

AGREE = 1e-11          # |mma - simt| / amp2
CASES = [              # N, M, S, D, kind
    (1, 127, 5, 1, "SE"),
    (63, 1, 1, 8, "ARDSE"),
    (64, 129, 40, 32, "Matern32"),
    (65, 10010, 5, 8, "Matern52"),
    (513, 127, 40, 1, "Matern32"),
    (513, 129, 3, 32, "ARDSE"),
    (2048, 10010, 5, 32, "Matern52"),
    (2048, 127, 40, 8, "SE"),
    (4097, 129, 1, 8, "ARDSE"),
    (4097, 1, 5, 32, "Matern52"),
    (8192, 10010, 1, 32, "Matern52"),
    (8192, 127, 1, 1, "Matern32"),
]


@pytest.fixture(scope="module")
def eng():
    import torch
    from spearmint_b200.engine import GPEIEngine
    return GPEIEngine(dtype=torch.float64)


def _inputs(eng, N, M, S, D, kind, seed):
    X, y, rs = data(N, D, seed)
    hs = synth_hypers(rs, S, D, 1e-3)
    C = np.vstack([X[:min(N, 3)], rs.rand(M, D)])[:M]         # candidates on the data first: var cancels there
    hb = eng.hypers(hs, kind)
    fac = eng.factor(kind, eng.to_dev(X), hb)
    fac.check_pd()
    alpha, _, _ = fac.solve(eng.to_dev(y), F=1)
    return dict(X=X, y=y, C=C, hs=hs, hb=hb, fac=fac, alpha=alpha.view(S, fac.Npad), Cd=eng.to_dev(C))


def _run(eng, name, P, M, ldm=None, ws_bytes=None, **over):
    import torch
    from spearmint_b200.engine import KINDS, ptr
    fac, hb = P["fac"], P["hb"]
    S = hb.S
    ldm = M + 3 if ldm is None else ldm
    mu = torch.full((S, ldm), float("nan"), dtype=torch.float64, device=eng.device)
    var = torch.full((S, ldm), float("nan"), dtype=torch.float64, device=eng.device)
    nb = lib().smk_predict_workspace_bytes(8, fac.Npad) if ws_bytes is None else ws_bytes
    ws = torch.empty((max(nb, 1),), dtype=torch.uint8, device=eng.device)
    a = dict(kind=KINDS[over.get("kind_name", fac.kind)], N=fac.N, Npad=fac.Npad, M=M, D=fac.D, S=S, X=ptr(fac.X),
             C=ptr(P["Cd"]), inv_ls=ptr(hb.inv_ls), amp2=ptr(hb.amp2), mean=ptr(hb.mean), L=ptr(fac.L),
             winv=ptr(fac.winv), alpha=ptr(P["alpha"]), mu=ptr(mu), var=ptr(var), ldm=ldm, ws=ptr(ws), nb=nb)
    a.update({k: v for k, v in over.items() if k != "kind_name"})
    rc = getattr(lib(), name)(a["kind"], a["N"], a["Npad"], a["M"], a["D"], a["S"], a["X"], a["C"], a["inv_ls"],
                              a["amp2"], a["mean"], a["L"], a["winv"], a["alpha"], a["mu"], a["var"], a["ldm"], a["ws"],
                              a["nb"], cur_stream())
    return rc, mu.cpu().numpy(), var.cpu().numpy()


@gpu
@pytest.mark.parametrize("N,M,S,D,kind", [pytest.param(*c, id="N%d-M%d-S%d-D%d-%s" % c) for c in CASES])
def test_predict_mma_matches_simt_and_oracle(eng, record_property, N, M, S, D, kind):
    """mu and var of the DMMA kernel against the SIMT kernel (1e-11 amp2) and the oracle (no further from it than the
    SIMT kernel, + 1e-11 amp2).  Worst |mma - simt| / amp2 measured on an H100 80GB HBM3 (SXM, 700 W power limit) over
    these cases: mu 5.2e-12 (N = 8192, D = 1), var 2.4e-15."""
    from oracle import gp_oracle as O
    P = _inputs(eng, N, M, S, D, kind, seed=N + 7 * M + S)
    rc1, mu1, var1 = _run(eng, "smk_predict_mma_f64", P, M)
    rc0, mu0, var0 = _run(eng, "smk_predict_f64", P, M)
    assert rc1 == 0 and rc0 == 0
    assert np.all(np.isfinite(mu1[:, :M])) and np.all(np.isfinite(var1[:, :M])), "unwritten entries j < M"
    assert np.all(np.isnan(mu1[:, M:])) and np.all(np.isnan(var1[:, M:])), "entries j >= M written (ldm = M + 3)"
    amp2 = P["hb"].host_amp2[:, None]
    dmu = float((np.abs(mu1[:, :M] - mu0[:, :M]) / amp2).max())
    dvar = float((np.abs(var1[:, :M] - var0[:, :M]) / amp2).max())
    record_property("mma_vs_simt_mu", dmu)
    record_property("mma_vs_simt_var", dvar)
    print("N=%d M=%d S=%d D=%d %s: max|dmu|/amp2 %.3e  max|dvar|/amp2 %.3e" % (N, M, S, D, kind, dmu, dvar))
    assert dmu <= AGREE and dvar <= AGREE, (dmu, dvar)
    if N > 2048:                       # the oracle's dense N x N solve per sample: small and medium N only
        return
    sub = np.arange(min(M, 300))
    for s in range(min(S, 3)):
        m, v, _, _ = O.predict(kind, P["hs"][s], P["X"], P["C"][sub], P["y"])
        a2 = P["hs"][s][2]
        for got, ref_simt, ref in ((mu1[s, sub], mu0[s, sub], m), (var1[s, sub], var0[s, sub], v)):
            e_mma, e_simt = np.abs(got - ref).max(), np.abs(ref_simt - ref).max()
            assert e_mma <= 2.0 * e_simt + AGREE * a2, (s, e_mma, e_simt)


@gpu
def test_predict_mma_argument_codes(eng):
    """The documented negative codes, in the order smk_predict_f64 checks them (header section 4 / 4-mma)."""
    P = _inputs(eng, 100, 50, 2, 3, "Matern52", seed=3)
    nb = lib().smk_predict_workspace_bytes(8, P["fac"].Npad)
    f = "smk_predict_mma_f64"
    assert _run(eng, f, P, 50)[0] == 0
    assert _run(eng, f, P, 50, kind=4)[0] == -1
    assert _run(eng, f, P, 50, kind=-1)[0] == -1
    assert _run(eng, f, P, 50, N=0)[0] == -2
    assert _run(eng, f, P, 50, Npad=100)[0] == -3
    assert _run(eng, f, P, 50, Npad=64)[0] == -3
    assert _run(eng, f, P, 0)[0] == -4
    assert _run(eng, f, P, 50, D=0)[0] == -5
    assert _run(eng, f, P, 50, S=0)[0] == -6
    for k in ("X", "C", "inv_ls", "amp2", "mean", "L", "winv", "alpha"):
        assert _run(eng, f, P, 50, **{k: None})[0] == -7, k
    assert _run(eng, f, P, 50, mu=None)[0] == -15
    assert _run(eng, f, P, 50, var=None)[0] == -15
    assert _run(eng, f, P, 50, ldm=49)[0] == -17
    assert _run(eng, f, P, 50, ws=None)[0] == -18
    # one work item (a single 64-candidate tile of one sample) needs one CTA's slab: 64 x Npad doubles
    assert _run(eng, f, P, 50, S=1, nb=64 * P["fac"].Npad * 8 - 8)[0] == -18
    assert _run(eng, f, P, 50, S=1, nb=64 * P["fac"].Npad * 8)[0] == 0
    assert nb >= 64 * P["fac"].Npad * 8


@gpu
def test_engine_routes_float64_predict_by_threshold(eng, monkeypatch):
    """GPEIEngine.predict on the float64 engine: N >= f64_mma_min_n runs smk_predict_mma_f64, smaller N smk_predict_f64;
    the float32 engine never does.  Both sides give the same moments (1e-11 amp2)."""
    import torch
    from spearmint_b200.engine import GPEIEngine
    P = _inputs(eng, 300, 500, 3, 4, "Matern52", seed=11)
    L = lib()
    outs = {}
    saved = eng.f64_mma_min_n
    try:
        for side, thr in (("mma", 300), ("simt", 301)):
            eng.f64_mma_min_n = thr
            assert eng.predict_kernel_for(300) == side
            n0 = L.smk_launch_count()
            mu, var, ldm = eng.predict("Matern52", P["fac"], P["Cd"], P["alpha"])
            torch.cuda.synchronize()
            assert L.smk_launch_count() - n0 == 1
            outs[side] = (mu[:, :500].cpu().numpy(), var[:, :500].cpu().numpy())
    finally:
        eng.f64_mma_min_n = saved
    a2 = P["hb"].host_amp2[:, None]
    for k in range(2):
        assert np.abs(outs["mma"][k] - outs["simt"][k]).max() / a2.min() <= AGREE
    assert GPEIEngine(dtype=torch.float32).predict_kernel_for(10 ** 6) == "simt"
    monkeypatch.setenv("SMK_F64_MMA_MIN_N", "77")
    assert GPEIEngine(dtype=torch.float64).f64_mma_min_n == 77
