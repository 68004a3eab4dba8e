"""CPU experiment: can the variance contraction beta = Linv @ Kx run as 3 x FP16 tensor products (hi*hi + hi*lo + lo*hi)
instead of 3 x TF32?  fp16 has tf32's 11-bit significand but only 5 exponent bits, so each operand is first multiplied by
an exact power of two that puts its largest |entry| in [2^14, 2^15); numpy float16 reproduces the round-to-nearest,
subnormal and overflow behaviour of the hardware conversion.  Products are exact and accumulated in float64 here (the
tensor core accumulates in fp32; that part is common to every variant and is covered by the fp32in row)."""
import os, sys
import numpy as np, scipy.linalg as spla
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import gp_oracle as O

def pow2_scale(x):
    m = np.abs(x).max()
    e = np.frexp(np.float32(m) * np.float32(1.00001))[1]      # m*1.00001 < 2^e
    return 15 - int(e)

def split16(x32):
    hi = x32.astype(np.float16)
    lo = (x32 - hi.astype(np.float32)).astype(np.float16)
    return hi.astype(np.float64), lo.astype(np.float64)

def trunc_tf32(x32):
    hi = (x32.view(np.uint32) & np.uint32(0xffffe000)).view(np.float32)
    lo = (x32 - hi)
    lo_hi = (lo.view(np.uint32) & np.uint32(0xffffe000)).view(np.float32)
    return hi.astype(np.float64), lo_hi.astype(np.float64)

def run(D, N, M, noise, kind='Matern52', seed=0, lsr=(0.3, 2.0), amp2=1.0):
    rs = np.random.RandomState(seed)
    X = rs.rand(N, D); C = rs.rand(M, D); C[:10] = X[0] + 1e-3 * rs.randn(10, D)
    y = np.sin(3 * X).sum(1); y = (y - y.mean()) / y.std()
    h = (0.0, noise, amp2, rs.uniform(*lsr, size=D))
    m, v, L, alpha = O.predict(kind, h, X, C, y)
    Kx = O.cov(kind, h[2], h[3], X, C)
    Linv = spla.solve_triangular(L, np.eye(N), lower=True)
    best = y.min()
    ei = O._ei_from_moments(best, m, np.sqrt(v))
    A32 = Linv.astype(np.float32); B32 = Kx.astype(np.float32)
    out = {}
    def report(name, beta):
        v2 = h[2] * (1 + 1e-6) - np.sum(beta.astype(np.float32).astype(np.float64) ** 2, axis=0)
        ei2 = O._ei_from_moments(best, m, np.sqrt(np.maximum(v2, 1e-300)))
        out[name] = (np.abs(v2 - v).max(), np.abs(ei2 - ei).max() / ei.max(), int(np.argmax(ei2) == np.argmax(ei)), int((v2 <= 0).sum()))
    report('fp32in', A32.astype(np.float64) @ B32.astype(np.float64))
    ah, al = trunc_tf32(A32); bh, bl = trunc_tf32(B32)
    report('3xtf32', ah @ bh + ah @ bl + al @ bh)
    ka, kb = pow2_scale(A32), pow2_scale(B32)
    As = np.ldexp(A32, ka); Bs = np.ldexp(B32, kb)
    ah, al = split16(As); bh, bl = split16(Bs)
    assert np.isfinite(ah).all() and np.isfinite(bh).all()
    report('3xfp16', np.ldexp(ah @ bh + ah @ bl + al @ bh, -(ka + kb)))
    # no scaling at all (what goes wrong without it)
    ah, al = split16(A32); bh, bl = split16(B32)
    report('3xfp16_unscaled', ah @ bh + ah @ bl + al @ bh)
    dyn = np.abs(A32[np.tril_indices(N)]); dyn = dyn[dyn > 0]
    return v.min(), (np.abs(A32).max(), np.quantile(dyn, 0.01)), out

if __name__ == '__main__':
    for cfg in [(2, 200, 2000, 1e-3), (8, 512, 3000, 1e-3), (8, 512, 3000, 1e-6), (20, 1024, 3000, 1e-3), (4, 1024, 3000, 1e-3),
                (32, 1500, 2000, 1e-3), (4, 1024, 3000, 1e-6), (8, 512, 3000, 1e-3, 'Matern52', 0, (0.3, 2.0), 37.0),
                (8, 512, 3000, 1e-3, 'Matern52', 0, (0.3, 2.0), 0.004), (6, 800, 2000, 1e-4, 'ARDSE'), (3, 600, 2000, 1e-2, 'Matern32')]:
        vmin, (amax, q01), res = run(*cfg)
        print(cfg, 'vmin %.2e  max|Linv| %.2e  1%%-quantile %.2e' % (vmin, amax, q01))
        for k, (dv, dei, am, neg) in res.items():
            print('   %-16s max|dv| %.2e  max|dEI|/maxEI %.2e argmax_ok %d neg %d' % (k, dv, dei, am, neg))
