import sys, time
sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__))))
import numpy as np, torch
import gnn_pathplanning_b200 as gp
from gnn_pathplanning_b200 import _lib, synthetic
from oracle import planner_oracle as po
class Cfg:
    num_agents, nGraphFilterTaps, device = 10, 3, torch.device("cuda")
sd = po.init_state_dict(3, seed=1); po.randomize_bn_stats(sd)
m = gp.DecentralPlannerNet(Cfg()); m.load_state_dict(sd); m = m.cuda().eval()
xs, Ss = [], []
for i in range(4):
    x, S = synthetic.make_batch(64, 10, 20, seed=10 + i)
    xs.append(torch.from_numpy(x).pin_memory()); Ss.append(torch.from_numpy(S).pin_memory())
outs = [torch.empty(10, 64, 5).pin_memory() for _ in range(8)]
def run(depth, steps=4000):
    tk = []
    t0 = None
    for i in range(steps + 50):
        if i == 50:
            for t in tk: m.wait(t)
            tk = []
            torch.cuda.synchronize(); t0 = time.perf_counter()
        if len(tk) >= depth:
            m.wait(tk.pop(0))
        tk.append(m.infer_host_async(xs[i % 4], Ss[i % 4], outs[i % 8]))
    for t in tk: m.wait(t)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e6
for lanes in (3, 4):
  _lib.set_debug_option("lanes", lanes)
  print("compute lanes:", lanes, flush=True)
  for mode in (0,):          # staging: 0 = copy engine (default), 1 = the 17 x 256-thread copy kernel
    _lib.set_debug_option("stage_mode", mode)
    for depth in (6, 8):
        us = run(depth)
        print("stage_mode=%d depth=%d: %.1f us/step  %.2f M agent-steps/s  (H2D %.1f GB/s)" % (mode, depth, us, 640 / us, 954880 / us * 1e-3), flush=True)
