"""The operand-precision model behind the tensor-core kernels, as executable checks on the CPU (numpy float16 reproduces
the hardware's round-to-nearest, subnormal and range behaviour; products exact, as on the tensor cores):

* the predict GEMM's scaled 3 x FP16 split is at least as accurate as the truncating 3 x TF32 split it replaced
  (DESIGN.md section 6, tools/fp16_split_experiment.py), also when amp2 is far from 1;
* the exact power-of-two scaling keeps every operand inside the fp16 range;
* the sample-factored distance  r2_s = sum_d w_sd (x_d - c_d)^2  evaluated as split products is as accurate as the
  float32 FMA chain (tools/kxt_tc_precision_experiment.py)."""
import numpy as np
import pytest
import scipy.linalg as spla

from oracle import gp_oracle as O


def _scale_exp(m):
    return 15 - int(np.frexp(np.float32(m) * np.float32(1.00001))[1])


def _split16(x32):
    hi = x32.astype(np.float16)
    lo = (x32 - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float64), lo.astype(np.float64)


def _trunc_tf32(x32):
    hi = (x32.view(np.uint32) & np.uint32(0xffffe000)).view(np.float32)
    lo = x32 - hi
    lo = (lo.view(np.uint32) & np.uint32(0xffffe000)).view(np.float32)
    return hi.astype(np.float64), lo.astype(np.float64)


@pytest.mark.parametrize("D,N,noise,amp2", [(2, 150, 1e-3, 1.0), (4, 300, 1e-6, 1.0), (6, 200, 1e-3, 37.0), (6, 200, 1e-4, 4e-3)])
def test_scaled_fp16_split_is_not_worse_than_tf32_split(D, N, noise, amp2):
    rs = np.random.RandomState(1)
    X, C = rs.rand(N, D), rs.rand(400, D)
    y = np.sin(3 * X).sum(1)
    h = (0.0, noise, amp2, rs.uniform(0.3, 2.0, D))
    m, v, L, _ = O.predict("Matern52", h, X, C, y)
    Kx = O.cov("Matern52", h[2], h[3], X, C)
    Linv = spla.solve_triangular(L, np.eye(N), lower=True)
    A32, B32 = Linv.astype(np.float32), Kx.astype(np.float32)

    def var_err(beta):
        return np.abs(h[2] * (1 + 1e-6) - np.sum(beta.astype(np.float32).astype(np.float64) ** 2, axis=0) - v).max()

    ah, al = _trunc_tf32(A32)
    bh, bl = _trunc_tf32(B32)
    e_tf32 = var_err(ah @ bh + ah @ bl + al @ bh)
    ka, kb = _scale_exp(np.abs(A32).max()), _scale_exp(np.abs(B32).max())
    As, Bs = np.ldexp(A32, ka), np.ldexp(B32, kb)
    lo_bound = 2.0 ** 14 / 1.0001                     # the 1.00001 safety factor can push a maximum just below 2^14
    assert lo_bound <= np.abs(As).max() < 2.0 ** 15 and lo_bound <= np.abs(Bs).max() < 2.0 ** 15
    ah, al = _split16(As)
    bh, bl = _split16(Bs)
    assert np.isfinite(ah).all() and np.isfinite(bh).all()
    e_fp16 = var_err(np.ldexp(ah @ bh + ah @ bl + al @ bh, -(ka + kb)))
    e_f32 = var_err(A32.astype(np.float64) @ B32.astype(np.float64))
    assert e_fp16 <= 1.05 * e_tf32 + 1e-12
    assert e_fp16 <= 8 * e_f32 + 1e-9 * amp2          # within a small factor of plain float32 operands


def test_sample_factored_distance_matches_fma_chain():
    rs = np.random.RandomState(0)
    D, N, M = 16, 256, 128
    X, C = rs.rand(N, D), rs.rand(M, D)
    C[:5] = X[0] + 1e-3 * rs.randn(5, D)
    ls = rs.uniform(0.3, 2.0, D)
    r2_64 = ((X[None] - C[:, None]) ** 2) @ (1.0 / ls ** 2)
    x32, c32, ils = X.astype(np.float32), C.astype(np.float32), (1.0 / ls).astype(np.float32)
    df = x32[None] * ils - c32[:, None] * ils
    r2_chain = np.zeros((M, N), np.float32)
    for d in range(D):
        r2_chain = r2_chain + df[..., d] * df[..., d]
    eq = _scale_exp((np.abs(x32).max() + np.abs(c32).max()) ** 2) & ~1
    hs = np.float32(2.0 ** (eq // 2))
    q32 = ((x32 * hs)[None] - (c32 * hs)[:, None]) ** 2
    w32 = ils * ils
    ew = _scale_exp(w32.max())
    qh, ql = (a.astype(np.float32) for a in _split16(q32))
    wh, wl = (a.astype(np.float32) for a in _split16(w32 * np.float32(2.0 ** ew)))
    assert np.isfinite(qh).all() and qh.max() < 2.0 ** 15
    acc = (ql @ wh).astype(np.float32) + (qh @ wl).astype(np.float32) + (qh @ wh).astype(np.float32)
    r2_tc = acc * np.float32(2.0 ** -(eq + ew))
    rel = lambda a: (np.abs(a.astype(np.float64) - r2_64) / r2_64)
    assert rel(r2_tc).mean() <= 1.5 * rel(r2_chain).mean() + 1e-9
    assert rel(r2_tc).max() <= 2.0 * rel(r2_chain).max() + 1e-7
    assert (r2_tc >= -1e-6).all()
