"""Per-layer phase timers of feature_mma_kernel ("tc_timing" debug option; thread 0 of block 0, i.e. the first warp of
warpgroup 0), in cycles per tile: waiting for filter chunks [6..11], issuing + waiting for the MMAs [12..17], input
conversion [19] and epilogues [26..31].  conv0 works from its accumulator fragments, so its MMAs are in its epilogue
column.
usage: python profiles/fm_phase_timing.py [episodes ...]   (10 agents per episode; default 64 4096 = 640 / 40,960 agents)"""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import gnn_pathplanning_b200 as gp
from gnn_pathplanning_b200 import _lib, synthetic
from oracle import planner_oracle as po


class Cfg:
    num_agents, nGraphFilterTaps, device = 10, 3, torch.device("cuda")


sd = po.init_state_dict(3, seed=1)
po.randomize_bn_stats(sd)
m = gp.DecentralPlannerNet(Cfg())
m.load_state_dict(sd)
m = m.cuda().eval()
m.set_feature_mode("mma")
_lib.set_debug_option("tc_timing", 1)
lib = _lib.load()
out = (C.c_ulonglong * 40)()
x, S = synthetic.make_batch(64, 10, 20, seed=3)
for B in [int(a) for a in sys.argv[1:]] or [64, 4096]:
    reps = (B + 63) // 64
    xt = torch.from_numpy(x).repeat(reps, 1, 1, 1, 1)[:B].cuda()
    St = torch.from_numpy(S).repeat(reps, 1, 1)[:B].cuda()
    with torch.no_grad():
        for _ in range(3):
            m.addGSO(St); m(xt)
        _lib.check(lib.gpp_debug_feature_mma_timing(out))      # drop the warm-up totals
        runs = 5
        for _ in range(runs):
            m.addGSO(St); m(xt)
        _lib.check(lib.gpp_debug_feature_mma_timing(out))
    v = list(out)
    t = max(v[18], 1)
    print("agents=%d  tiles timed (block 0, %d launches) %d" % (B * 10, runs, t))
    print("  layer   filter-wait       mma  epilogue   (cycles per tile)")
    tot = 0.0
    for L in range(6):
        w, mm, e = v[6 + L] / t, v[12 + L] / t, v[26 + L] / t
        if L == 0:      # conv0's timer [26] runs from before its filter wait: MMAs + fragment epilogue, wait taken out
            e -= w
        tot += w + mm + e
        print("  %-6s %11.0f %9.0f %9.0f" % (["conv0", "conv1", "conv2", "conv3", "conv4", "linear"][L], w, mm, e))
    print("  input conversion %.0f; sum %.0f cycles per tile (%.1f us at 1.98 GHz)" % (v[19] / t, tot + v[19] / t,
                                                                                     (tot + v[19] / t) / 1980.0))
