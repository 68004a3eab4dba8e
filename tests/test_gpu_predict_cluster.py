"""The predict GEMM (predict_tc_kernel modes 0 and 1) runs in 2-CTA clusters: the CTAs of a cluster hold adjacent
candidate tiles of the same (sample, row-group pair) and share every Linv / alpha^T tile through TMA multicast.  These
cases reach the cluster's edges: one tile (the partner has no tile of its own), odd tile counts (the partner of the last
cluster re-runs the last tile and writes nothing), odd and even row-group counts (the middle group of an odd count is
skipped by both CTAs), S = 1 and S = 40, fantasies (mode 1) and a chunked call whose chunks have odd and even tile counts.

Every stage is checked against float64 at the bounds of tests/test_gpu_predict.py (_tc_stages), and a second call must
give the same bits.
"""
import numpy as np
import pytest

from tests.helpers import Worst, same as _same
from tests.test_gpu_predict import _alpha_f, _cands, _predict_tc, _setup, _subset, _tc_stages, engs  # noqa: F401

gpu = pytest.mark.gpu


def _again(P, Cd, F, af_dev, r):
    r2 = _predict_tc(P, Cd, F=F, alpha_f=af_dev, dbg=True)
    for k in ("mu", "var", "mu_f", "dbg"):
        if k in r:
            assert _same(r2[k], r[k]), "%s: a second call differs" % k


@gpu
@pytest.mark.parametrize("N,S,M,F", [
    pytest.param(255, 1, 128, 1, id="g1-N255-S1-tiles1"),
    pytest.param(511, 2, 256, 100, id="g2-N511-S2-tiles2-F100"),
    pytest.param(767, 3, 384, 257, id="g3-N767-S3-tiles3-F257"),
    pytest.param(768, 1, 385, 1, id="g3-N768-S1-tiles4-ragged"),
    pytest.param(1024, 40, 640, 2, id="g4-N1024-S40-tiles5-F2"),
])
def test_predict_cluster_tile_counts(engs, record_property, N, S, M, F):  # noqa: F811
    P = _setup(engs, "tc", "Matern52", N, 8, 1e-3, S, seed=N + S)
    C, Cd = _cands(P, M, seed=N + 11)
    af_dev, af = (None, None) if F == 1 else _alpha_f(P, F, seed=N + 12)
    W = Worst(record_property)
    sub = np.arange(M) if M <= 400 else _subset(M, P["rs"])
    r, _ = _tc_stages(W, P, C, Cd, sub, F, af_dev, af, samples=None if S <= 3 else (0, S - 1))
    _again(P, Cd, F, af_dev, r)
    W.flush()


@gpu
def test_predict_cluster_chunks_odd_and_even_tiles(engs, record_property, monkeypatch):  # noqa: F811
    """A 4 MB budget at N = 1024, S = 2 gives chunks of 512 candidates (4 tiles).  M = 1700 leaves a tail of 164
    candidates (2 tiles, one ragged), M = 1400 a tail of 376 (3 tiles: the last cluster has one CTA without a tile).
    Chunked results equal the single-chunk call bit for bit."""
    P = _setup(engs, "tc", "Matern52", 1024, 8, 1e-3, 2, seed=5)
    for M in (1700, 1400):
        C, Cd = _cands(P, M, seed=M)
        af_dev, af = _alpha_f(P, 3, seed=M + 1)
        one = _predict_tc(P, Cd, F=3, alpha_f=af_dev, dbg=True)
        monkeypatch.setenv("SMK_TC_BUDGET_MB", "4")
        many = _predict_tc(P, Cd, F=3, alpha_f=af_dev)
        monkeypatch.delenv("SMK_TC_BUDGET_MB")
        for k in ("mu", "var", "mu_f"):
            assert _same(many[k], one[k]), "M = %d, %s: chunked differs from one chunk" % (M, k)
        W = Worst(record_property)
        _tc_stages(W, P, C, Cd, _subset(M, P["rs"], chunk=512, extra=100), 3, af_dev, af, r=one)
        W.flush()
