"""Throughput of the device-resident expert dataset (gnn_pathplanning_b200.ExpertDataset, csrc/expert_data.cu) next to
the reference's way of feeding training: the transform to one .mat file per case and a loader that opens one file
per sample.  Prints the GPU's name and power limit with the numbers.

  transform   add_cases (host padding, one copy, gpp_expert_radius) + every sample gathered once (gpp_expert_gather),
              for C synthetic cases, against oracle/expert_data_oracle.transform (the reference's algorithm) on one core
  batch()     one minibatch of 64 samples (x, one-hot target, f32 GSO) gathered on the device
  .mat loader the reference loader's work per batch of 64 samples: scipy.io.loadmat of 64 files written by
              scipy.io.savemat with the transformer's fields, sliced to one step each (load_train_data)
usage: python profiles/expert_data_throughput.py [cases] [agents] [map_w]"""
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import scipy.io as sio
import torch

import gnn_pathplanning_b200 as gp
from gnn_pathplanning_b200 import synthetic
from oracle import expert_data_oracle as edo


def make_cases(C, N, W, seed=1):
    """Random maps, starts and goals; each agent walks along x, then along y (obstacles ignored: the transform does
    not look at them)."""
    rng = np.random.default_rng(seed)
    maps, goals, paths, makespans = [], [], [], []
    for _ in range(C):
        m, start, goal = synthetic.random_episode(rng, N, W, 0.1)
        ps = []
        for (sx, sy), (gx, gy) in zip(start.tolist(), goal.tolist()):
            stepx = 1 if gx >= sx else -1
            stepy = 1 if gy >= sy else -1
            p = [(x, sy) for x in range(sx, gx + stepx, stepx)] + [(gx, y) for y in range(sy + stepy, gy + stepy, stepy)]
            ps.append(p)
        maps.append(m.astype(np.uint8))
        goals.append(goal)
        paths.append(ps)
        makespans.append(max(len(p) for p in ps) - 1)
    return np.stack(maps), np.stack(goals), paths, np.array(makespans)


def cuda_ms(fn, reps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    torch.cuda.synchronize()
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def main():
    C = int(sys.argv[1]) if len(sys.argv) > 1 else 21000
    N = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    W = int(sys.argv[3]) if len(sys.argv) > 3 else 20
    assert torch.cuda.is_available(), "expert_data_throughput measures on a CUDA device"
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True).stdout.strip()
    except OSError:
        power = "unknown"
    maps, goals, paths, makespans = make_cases(C, N, W)
    gp.ExpertDataset(N, W).add_cases(maps[:16], goals[:16], paths[:16], makespans[:16])        # warm-up
    times = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ds = gp.ExpertDataset(N, W)
        ds.add_cases(maps, goals, paths, makespans)
        t_add = time.perf_counter() - t0
        for lo in range(0, len(ds), 8192):
            ds._gather(torch.arange(lo, min(lo + 8192, len(ds)), device="cuda"))
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0, t_add))
    t_all, t_add = min(times)
    R = len(ds)
    ms_radius = cuda_ms(lambda: gp._lib.check(ds.lib.gpp_expert_radius(
        ds.states.data_ptr(), ds.case_offset.data_ptr(), ds.case_steps.data_ptr(), ds.goal.data_ptr(), 5.0,
        torch.empty(C, device="cuda", dtype=torch.float64).data_ptr(), torch.empty(C, device="cuda", dtype=torch.int32).data_ptr(),
        torch.empty(C, 2, device="cuda", dtype=torch.int32).data_ptr(), C, N, ds._stream())), 5)
    # the oracle transform on one core
    sub = min(100, C)
    t0 = time.process_time()
    for c in range(sub):
        edo.transform(maps[c], goals[c], paths[c], makespans[c])
    cpu_case = (time.process_time() - t0) / sub
    # one minibatch of 64 samples
    rows = torch.randperm(R, device="cuda")[:64]
    us_gather = cuda_ms(lambda: ds._gather(rows), 2000) * 1e3          # back to back: bound by the host launch path
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(200):
            ds._gather(rows)
        torch.cuda.synchronize()
    k = [e for e in prof.key_averages() if "expert_gather_kernel" in e.key]
    us_kernel = k[0].device_time_total / k[0].count if k else float("nan")
    rows_h = rows.cpu().numpy()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(500):
        ds.batch(rows_h)
    torch.cuda.synchronize()
    us_batch = (time.perf_counter() - t0) / 500 * 1e6
    bytes_out = 64 * N * (3 * 11 * 11 * 4 + 5 * 8 + N * 4)
    # the reference loader: 64 .mat files, one sample each
    with tempfile.TemporaryDirectory() as tmp:
        files = []
        for c in range(64):
            d, _ = edo.transform(maps[c], goals[c], paths[c], makespans[c])
            path = os.path.join(tmp, "train_ID%05d_MP%d.mat" % (c, d["makespan"]))
            sio.savemat(path, d)
            files.append((path, c % d["makespan"]))
        reps = 5
        t0 = time.perf_counter()
        for _ in range(reps):
            for path, step in files:
                dc = sio.loadmat(path)
                torch.from_numpy(dc["inputTensor"][step][:]).float()
                torch.from_numpy(dc["GSO"][step, :, :]).float()
                torch.from_numpy(dc["target"][step, :, :]).long()
                torch.from_numpy(dc["map"]).float()
        ms_mat = (time.perf_counter() - t0) / reps * 1e3
    print("GPU: %s, power limit %s" % (name, power))
    print("transform: %d cases (N=%d, %dx%d, %d samples): add_cases %.3f s, + every sample gathered: %.3f s = "
          "%.0f cases/s, %.0f samples/s (radius kernel alone %.2f ms)" % (C, N, W, W, R, t_add, t_all, C / t_all,
                                                                          R / t_all, ms_radius))
    print("oracle transform (numpy, one CPU core): %.2f ms per case = %.0f cases/s" % (cpu_case * 1e3, 1 / cpu_case))
    print("batch of 64 x %d agents (%.2f MB written): gather kernel %.2f us on the device, %.2f us per call back to "
          "back (batches()), batch(numpy indices) incl. index check and copy %.1f us; training step 1.67 ms"
          % (N, bytes_out / 1e6, us_kernel, us_gather, us_batch))
    print(".mat loader (scipy.io.loadmat, CPU): %.1f ms per batch of 64 samples" % ms_mat)


if __name__ == "__main__":
    main()
