"""Per-phase cycles of block 0 of feature_kernel and gf_fwd_kernel inside the planner forward
("fe_timing" / "gf_timing" debug options)."""
import os, sys, ctypes as C
sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__))))
import torch
import gnn_pathplanning_b200 as gp
from gnn_pathplanning_b200 import _lib, synthetic

class Cfg:
    def __init__(self, n, k):
        self.num_agents, self.nGraphFilterTaps, self.device = n, k, torch.device("cuda")

names = ["prologue", "stage x/S", "propagate", "contract", "epilogue", "action+merge"]
lib = _lib.load()
_lib.set_debug_option("gf_timing", 1)
_lib.set_debug_option("fe_timing", 1)
for (B, N) in [(64, 10), (256, 10), (1024, 10), (64, 20)]:
    m = gp.DecentralPlannerNet(Cfg(N, 3)).cuda().eval()
    m.set_graph_filter_mode("cuda")
    x, S = synthetic.make_batch(B, N, 20, seed=1)
    xt, St = torch.from_numpy(x).cuda(), torch.from_numpy(S).cuda()
    m.addGSO(St)
    out = (C.c_ulonglong * 6)()
    fo = (C.c_ulonglong * 7)()
    m.set_feature_mode("cuda")
    with torch.no_grad():
        for _ in range(5):
            m(xt)
        lib.gpp_debug_gf_timing(out)
        lib.gpp_debug_feature_timing(fo)
        reps = 20
        for _ in range(reps):
            m(xt)
        lib.gpp_debug_gf_timing(out)
        lib.gpp_debug_feature_timing(fo)
    fn = ["stage", "conv0", "conv1", "conv2", "conv3", "conv4", "mlp+store"]
    fv = [o / reps for o in fo]
    print("B=%d N=%d  feature_kernel block 0: " % (B, N) + "  ".join("%s %.0f" % (n, c) for n, c in zip(fn, fv)) + "  total %.0f cycles" % sum(fv))
    v = [o / reps for o in out]
    print("B=%d N=%d  " % (B, N) + "  ".join("%s %.0f" % (n, c) for n, c in zip(names, v)) + "  total %.0f cycles" % sum(v))
