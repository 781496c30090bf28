"""Throughput of expert case generation (gnn_pathplanning_b200.generate_cases, csrc/case_gen.cu) next to the oracle
(oracle/case_gen_oracle.py, the same contract in numpy / Python) on one CPU core.  Prints the GPU's name and power
limit with the numbers.

  accepted cases/s of generate_cases (wall time from the call to its return, which waits for the device: the kernel,
    the compaction and the copies; best of 3 after a warm-up), at the reference's density 0.1 and complexity 0.01:
    100,000 cases at N = 10 on 20x20 maps and 20,000 at N = 64 on 64x64;
  the kernel alone: CUDA events around one gpp_case_generate call over the same candidates;
  the oracle's accepted cases/s on one CPU core;
  generation as a share of generate + solve: generate_cases then solve_cases (H = 256, 2,048 nodes) of 4,096 cases.
usage: python profiles/case_gen_throughput.py"""
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import gnn_pathplanning_b200 as gp
from gnn_pathplanning_b200 import _lib
from oracle import case_gen_oracle as cgo


def wall(fn, reps=3):
    fn()
    best, out = None, None
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    return best, out


def kernel_ms(K, N, W):
    aisles, walk = cgo.sizes(W, 0.1, 0.01)
    m = torch.empty(K, W, W, device="cuda", dtype=torch.uint8)
    s, g = (torch.empty(K, N, 2, device="cuda", dtype=torch.int32) for _ in range(2))
    st = torch.empty(K, device="cuda", dtype=torch.int32)
    lib, stream = _lib.load(), torch.cuda.current_stream().cuda_stream
    call = lambda: _lib.check(lib.gpp_case_generate(1337, 0, K, N, W, aisles, walk, m.data_ptr(), s.data_ptr(),
                                                    g.data_ptr(), st.data_ptr(), stream))
    call()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        call()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 5


def throughput(C, N, W, oracle_candidates):
    dt, res = wall(lambda: gp.generate_cases(C, N, W))
    K = int(res.candidate[-1]) + 1
    ms = kernel_ms(K, N, W)
    t0 = time.process_time()
    o = cgo.candidates(1337, 0, oracle_candidates, N, W)
    cpu = time.process_time() - t0
    acc = int((o["status"] == cgo.ACCEPTED).sum())
    print("N=%d, %dx%d: %d cases from %d candidates (accepted %.3f, too few free %.3f, shared cell %.3f) in %.4f s = "
          "%.0f cases/s; kernel %.3f ms for the %d candidates = %.0f candidates/s; oracle (one CPU core) %.0f "
          "cases/s (%d candidates)" % (N, W, W, C, K, res.tallies["ACCEPTED"] / K, res.tallies["TOO_FEW_FREE"] / K,
                                      res.tallies["SHARED_CELL"] / K, dt, C / dt, ms, K, K / ms * 1e3, acc / cpu,
                                      oracle_candidates))


def share_of_solve(C, N, W):
    gen, cases = wall(lambda: gp.generate_cases(C, N, W))
    solve, res = wall(lambda: gp.solve_cases(cases.maps, cases.starts, cases.goals, ids=cases.ids))
    frac = np.bincount(res.status, minlength=3) / C
    print("N=%d, %dx%d, %d cases: generate %.4f s, solve %.4f s (solved %.3f); generation is %.2f %% of generate + "
          "solve" % (N, W, W, C, gen, solve, frac[0], 100 * gen / (gen + solve)))


def main():
    assert torch.cuda.is_available(), "case_gen_throughput measures on a CUDA device"
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True).stdout.strip()
    except OSError:
        power = "unknown"
    print("GPU: %s, power limit %s" % (torch.cuda.get_device_name(0), power))
    throughput(100_000, 10, 20, 4000)
    throughput(20_000, 64, 64, 200)
    share_of_solve(4096, 10, 20)


if __name__ == "__main__":
    main()
