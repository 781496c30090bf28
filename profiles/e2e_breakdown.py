"""Host-side cost of the pipelined host-buffer path at the headline size: time spent in infer_host_async
(submission) and in wait() per step, next to the device-only step time."""
import sys, time
sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__))))
import torch
import gnn_pathplanning_b200 as gp
from gnn_pathplanning_b200 import synthetic

class Cfg:
    def __init__(self, n, k):
        self.num_agents, self.nGraphFilterTaps, self.device = n, k, torch.device("cuda")

B, N, STEPS = 64, 10, 400
m = gp.DecentralPlannerNet(Cfg(N, 3)).cuda().eval()
pool = [synthetic.make_batch(B, N, 20, seed=s) for s in range(8)]
hx = [torch.from_numpy(x).pin_memory() for x, _ in pool]
hS = [torch.from_numpy(S).pin_memory() for _, S in pool]
for depth in (2, 3):
    outs = [torch.empty(N, B, 5).pin_memory() for _ in range(depth)]
    for i in range(20):
        m.wait(m.infer_host_async(hx[i % 8], hS[i % 8], outs[i % depth]))
    t_sub = t_wait = 0.0
    q = []
    t0 = time.perf_counter()
    for i in range(STEPS):
        a = time.perf_counter()
        q.append(m.infer_host_async(hx[i % 8], hS[i % 8], outs[i % depth]))
        b = time.perf_counter()
        t_sub += b - a
        if len(q) >= depth:
            m.wait(q.pop(0))
            t_wait += time.perf_counter() - b
    for t in q:
        m.wait(t)
    tot = time.perf_counter() - t0
    print("depth %d: %.1f us/step  (submit %.1f us, wait %.1f us)  %.2f M agent-steps/s"
          % (depth, tot / STEPS * 1e6, t_sub / STEPS * 1e6, t_wait / STEPS * 1e6, B * N * STEPS / tot / 1e6))
xd, Sd = torch.from_numpy(pool[0][0]).cuda(), torch.from_numpy(pool[0][1]).cuda()
m.addGSO(Sd)
with torch.no_grad():
    for _ in range(20):
        m(xd)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(STEPS):
        m(xd)
    torch.cuda.synchronize()
print("device-resident forward: %.1f us/step" % ((time.perf_counter() - t0) / STEPS * 1e6))
