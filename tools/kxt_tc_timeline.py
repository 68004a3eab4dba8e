"""Dumps the clock64() timeline of the tensor-core generator (first 64 tiles of CTA 0).  SMK_KXT_TIMELINE=1 must be set."""
import ctypes, os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["SMK_KXT_TIMELINE"] = "1"
from spearmint_b200 import _lib
from spearmint_b200.engine import GPEIEngine, ptr, check, KINDS
eng = GPEIEngine(device="cuda:0", dtype=torch.float32)
L = _lib.lib()
D, N, M, S = 32, 4096, 132 * 3 * 4, 40
rs = np.random.RandomState(0)
X, C = rs.rand(N, D), rs.rand(M, D)
hs = [(0.0, 1e-3, 1.0, rs.uniform(0.3, 2.0, D)) for _ in range(S)]
hb = eng.hypers(hs, "Matern52")
Np, Mc = L.smk_tc_np(N), ((M + 127) // 128) * 128
Xd, Cd = eng.to_dev(X), eng.to_dev(C)
alpha = torch.randn((S, Np), dtype=torch.float32, device=eng.device)
h16 = torch.empty((S, Mc, Np), dtype=torch.float16, device=eng.device); l16 = torch.empty_like(h16)
mu = torch.zeros((S, Mc), dtype=torch.float32, device=eng.device)
nb = L.smk_kxt_pack_workspace_bytes(Np, M, S); ws = torch.empty((nb,), dtype=torch.uint8, device=eng.device)
for it in range(2):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    check(L.smk_kxt_pack_f16(1, KINDS["Matern52"], N, Np, M, D, S, ptr(Xd), ptr(Cd), ptr(hb.inv_ls), ptr(hb.amp2), ptr(hb.mean),
                             ptr(alpha), Np, ptr(h16), ptr(l16), ptr(mu), Mc, ptr(ws), nb, eng.stream()), "kxt")
    ev1.record(); torch.cuda.synchronize()
    print("launch %d: %.3f ms for %d items x 32 tiles" % (it, ev0.elapsed_time(ev1), (Mc + 2) // 3))
out = (ctypes.c_longlong * 512)()
assert L.smk_debug_kxt_tc_timeline(out, 512) == 0
tl = np.array(out[:], dtype=np.int64).reshape(64, 8)[:, :4]
t0 = tl[0, 0]
print("tile  mma_issue  next_q_built  mma_done  epilogue_done   (cycles from first stamp)")
for t in range(40):
    print("%3d  " % t + " ".join("%9d" % (v - t0) for v in tl[t]))
print("tile period median", np.median(np.diff(tl[8:40, 0])), " q build median", np.median(tl[8:40, 1] - tl[8:40, 0]),
      " MMA wait after the build median", np.median(tl[8:40, 2] - tl[8:40, 1]), " epilogue median", np.median(tl[8:40, 3] - tl[8:40, 2]))
