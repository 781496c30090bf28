"""Feature extractor alone (events around the kernel inside the planner forward, programmatic launch off) and the
whole device-resident step (programmatic launch on), per feature kernel, over agent counts.
usage: python profiles/fe_microbench.py [agents ...]"""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import gnn_pathplanning_b200 as gp
from gnn_pathplanning_b200 import _lib, synthetic
from oracle import planner_oracle as po


class Cfg:
    def __init__(self, n, k):
        self.num_agents, self.nGraphFilterTaps, self.device = n, k, torch.device("cuda")


sizes = [int(a) for a in sys.argv[1:]] or [64, 100, 410, 1024, 4096]
N, K = 10, 3
sd = po.init_state_dict(K, seed=1)
po.randomize_bn_stats(sd)
for B in sizes:
    x, S = synthetic.make_batch(min(B, 64), N, 20, seed=3)
    reps = (B + x.shape[0] - 1) // x.shape[0]
    xt = torch.from_numpy(x).repeat(reps, 1, 1, 1, 1)[:B].cuda()
    St = torch.from_numpy(S).repeat(reps, 1, 1)[:B].cuda()
    for fe in ("cuda", "tc", "mma"):
        m = gp.DecentralPlannerNet(Cfg(N, K))
        m.load_state_dict(sd)
        m = m.cuda().eval()
        m.set_feature_mode(fe)
        iters = 300 if B * N < 20000 else 40
        with torch.no_grad():
            for _ in range(5):
                m.addGSO(St); m(xt)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                m.addGSO(St); m(xt)
            e1.record(); torch.cuda.synchronize()
            step_us = e0.elapsed_time(e1) * 1e3 / iters
            nat = m._native_for(xt.device)
            _lib.check(nat.lib.gpp_planner_set_profiling(nat.handle, 1))
            for _ in range(iters):
                m.addGSO(St); m(xt)
            fe_ms, gf_ms, nst = C.c_double(), C.c_double(), C.c_int()
            _lib.check(nat.lib.gpp_planner_get_profile(nat.handle, C.byref(fe_ms), C.byref(gf_ms), C.byref(nst)))
            _lib.check(nat.lib.gpp_planner_set_profiling(nat.handle, 0))
        fe_us = fe_ms.value * 1e3 / max(1, nst.value)
        print("agents=%6d  feature=%-4s  feature kernel %9.1f us (%6.0f cycles/agent/SM-slot)  filter %7.1f us  step %9.1f us  %7.2f M agent-steps/s"
              % (B * N, fe, fe_us, fe_us * 1980.0 / max(1.0, B * N / torch.cuda.get_device_properties(0).multi_processor_count), gf_ms.value * 1e3 / max(1, nst.value), step_us,
                 B * N / step_us), flush=True)
