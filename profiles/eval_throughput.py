"""Test cases evaluated per second by gnn_pathplanning_b200.evaluate (batched, device-resident rollouts + scoring), next
to the CPU time per case of the plain-Python simulator + scoring (oracle/eval_oracle.py, the reference's algorithm)
replaying the same logits.  Prints the GPU's name and power limit with the numbers.
usage: python profiles/eval_throughput.py [cases] [agents] [map_w]"""
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import gnn_pathplanning_b200 as gp
from gnn_pathplanning_b200 import synthetic
from oracle import eval_oracle, planner_oracle as po, sim_oracle


class Cfg:
    def __init__(self, n):
        self.num_agents, self.nGraphFilterTaps, self.device = n, 3, torch.device("cuda")
        self.rate_maxstep, self.commR = 2, 6


class Recording(torch.nn.Module):
    def __init__(self, inner):
        super().__init__()
        self.inner, self.logits = inner, []

    def addGSO(self, S):
        self.inner.addGSO(S)

    def forward_logits(self, x):
        out = self.inner.forward_logits(x)
        self.logits.append(out.cpu().numpy())
        return out


def make_cases(B, N, W, seed=1):
    rng = np.random.default_rng(seed)
    cases = []
    while len(cases) < B:
        m, start, goal = synthetic.random_episode(rng, N, W, 0.1)
        if not (start == goal).all(axis=1).any():
            c = eval_oracle.expert_case(m, start, goal)
            if c is not None:
                cases.append(c)
    return cases


def main():
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
    N = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    W = int(sys.argv[3]) if len(sys.argv) > 3 else 20
    assert torch.cuda.is_available(), "eval_throughput measures on a CUDA device"
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True).stdout.strip()
    except OSError:
        power = "unknown"
    cases = make_cases(B, N, W)
    sd = po.init_state_dict(3, seed=1)
    sd["actionsMLP.0.weight"] = sd["actionsMLP.0.weight"] * 40.0
    m = gp.DecentralPlannerNet(Cfg(N))
    m.load_state_dict(sd)
    m = m.cuda().eval()
    cfg = Cfg(N)
    gp.evaluate(m, cases[:256], cfg)                          # warm-up: module load, planner workspaces
    times = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = gp.evaluate(m, cases, cfg)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    t = min(times)
    # the CPU simulator + scoring on a subset, fed with the GPU planner's own logits (planner time not included)
    sub = cases[:64]
    rec = Recording(m)
    gp.evaluate(rec, sub, cfg)
    rate = 3 if N >= 20 else cfg.rate_maxstep
    t0 = time.process_time()
    for b, (inp, tgt, makespan, _, mp) in enumerate(sub):
        goal, start = inp[0, 0].int().numpy(), inp[0, 1].int().numpy()
        mt, ft, _ = eval_oracle.path_target(start, goal, tgt[0].argmax(-1).numpy())
        sim = sim_oracle.SimOracle(N, 6.0).setup(start, goal, mp[0].numpy(), int(makespan[0].int()) * rate)
        eval_oracle.policy_outcome(sim, lambda s: rec.logits[s][:, b], mt, ft)
    cpu_per_case = (time.process_time() - t0) / len(sub)
    print("GPU: %s, power limit %s" % (name, power))
    print("evaluate: %d cases, N=%d, %dx%d: %.3f s (best of %d) = %.0f cases/s; rateReachGoal %.4f"
          % (B, N, W, W, t, len(times), B / t, res.rateReachGoal))
    print("oracle simulator + scoring (CPU, logits given, no planner): %.2f ms per case" % (cpu_per_case * 1e3))


if __name__ == "__main__":
    main()
