"""Throughput of the batched expert solver (gnn_pathplanning_b200.solve_cases, csrc/expert_solve.cu) next to the
oracle (oracle/solver_oracle.py, the same contract in plain Python) on one CPU core.  Prints the GPU's name and power
limit with the numbers.  The reference's own solver (the prebuilt `ecbs` binary) is not measured here.

Two workloads of C cases at N agents on W x W maps:
  random    synthetic.random_episode: uniform starts and goals, 10 % obstacles
  failures  the failure cases of a random-weight planner: collect_failure_cases on test items of the random cases
            solved first (so the agents start where the planner left them)
For each: cases/s of solve_cases (wall time incl. copies, best of 3), the SOLVED / NO_SOLUTION / BUDGET fractions,
nodes created at the median and the maximum, and the oracle's cases/s on a subset.
usage: python profiles/solver_throughput.py [cases] [agents] [map_w]"""
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import gnn_pathplanning_b200 as gp
from gnn_pathplanning_b200 import synthetic
from oracle import planner_oracle as po
from oracle import solver_oracle as so

H, MAX_NODES, ORACLE_SUBSET = 256, 2048, 100


class Cfg:
    def __init__(self, n):
        self.num_agents, self.nGraphFilterTaps, self.device = n, 3, torch.device("cuda")
        self.rate_maxstep, self.commR = 2, 6


def random_cases(C, N, W, seed):
    rng = np.random.default_rng(seed)
    cases = [synthetic.random_episode(rng, N, W, 0.1) for _ in range(C)]
    return (np.stack([c[0] for c in cases]).astype(np.uint8), np.stack([c[1] for c in cases]),
            np.stack([c[2] for c in cases]))


def failure_cases(C, N, W):
    """Failure cases of a random-weight planner, drawn until there are C of them."""
    sd = po.init_state_dict(3, seed=3)
    m = gp.DecentralPlannerNet(Cfg(N))
    m.load_state_dict(sd)
    m = m.cuda().eval()
    maps, starts, goals = [], [], []
    seed = 100
    while sum(len(s) for s in starts) < C:
        maps_r, starts_r, goals_r = random_cases(2048, N, W, seed)
        moving = (starts_r != goals_r).any(-1).all(-1)     # the reference's test() cannot score an agent that never moves
        sol = gp.solve_cases(maps_r[moving], starts_r[moving], goals_r[moving]).solutions()
        seed += 1
        ds = gp.ExpertDataset(N, W)
        ds.add_cases(sol.maps, sol.goals, sol.paths, sol.makespans)
        _, fc = gp.collect_failure_cases(m, list(ds.test_cases()), Cfg(N))
        maps.append(fc.map)
        starts.append(fc.start.cpu().numpy())
        goals.append(fc.goal)
    return np.concatenate(maps)[:C], np.concatenate(starts)[:C], np.concatenate(goals)[:C]


def measure(name, maps, starts, goals):
    gp.solve_cases(maps[:64], starts[:64], goals[:64])         # warm-up
    best = None
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = gp.solve_cases(maps, starts, goals, max_makespan=H, max_nodes=MAX_NODES)
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    C = len(res)
    frac = np.bincount(res.status, minlength=3) / C
    t0 = time.process_time()
    want = so.solve_all(maps[:ORACLE_SUBSET], starts[:ORACLE_SUBSET], goals[:ORACLE_SUBSET], H, MAX_NODES)
    cpu = (time.process_time() - t0) / min(C, ORACLE_SUBSET)
    same = all(np.array_equal(want[k], getattr(res, m)[:ORACLE_SUBSET]) for k, m in
               (("status", "status"), ("created", "nodes_created"), ("paths", "paths")))
    print("%s: %d cases (N=%d, %dx%d, H=%d, max_nodes=%d): %.3f s = %.0f cases/s; solved %.3f, no solution %.3f, "
          "budget %.3f; nodes created median %d, max %d; oracle (one CPU core) %.1f cases/s on %d cases, matches: %s"
          % (name, C, starts.shape[1], maps.shape[1], maps.shape[1], H, MAX_NODES, best, C / best, frac[0], frac[1],
             frac[2], int(np.median(res.nodes_created)), int(res.nodes_created.max()), 1 / cpu,
             min(C, ORACLE_SUBSET), same))


def main():
    C = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
    N = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    W = int(sys.argv[3]) if len(sys.argv) > 3 else 20
    assert torch.cuda.is_available(), "solver_throughput measures on a CUDA device"
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True).stdout.strip()
    except OSError:
        power = "unknown"
    print("GPU: %s, power limit %s" % (name, power))
    measure("random", *random_cases(C, N, W, 1))
    measure("failures", *failure_cases(C, N, W))


if __name__ == "__main__":
    main()
