"""Graph-filter kernel micro-benchmark (device-resident, CUDA events): CUDA-core vs tensor-core (wgmma) kernels over
batch sizes, reported as agent-steps/s and as algorithmic GB/s (SURVEY.md 8d: 4*(G+N+F) bytes per
agent-step) against the measured HBM peak (else the H100 SXM data-sheet figure).  usage: python profiles/gf_microbench.py [N] [K] [modes, e.g. 3 or 1,2,3]"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CHILD = r'''
import sys, json, torch
sys.path.insert(0, %r)
import gnn_pathplanning_b200 as gp
N, K = int(sys.argv[1]), int(sys.argv[2])
from gnn_pathplanning_b200 import _lib
_lib.set_debug_option("gf_mode", int(sys.argv[3]))
torch.manual_seed(0)
w = ((torch.rand(128, 1, K, 128) - 0.5) * 0.2).cuda()
b = (torch.rand(128, 1) - 0.5).cuda()
out = []
for B in (64, 512, 4096, 32768, 131072):
    x = torch.randn(B, N, 128, device="cuda")
    # rollout-like GSO: normalised adjacency of random agent positions on a 20x20 map, radius 6
    pos = torch.randint(0, 20, (B, N, 2), device="cuda").float()
    A = ((pos[:, :, None, :] - pos[:, None, :, :]).norm(dim=-1) < 6.0).float() * (1.0 - torch.eye(N, device="cuda"))
    dinv = A.sum(-1).clamp(min=1.0).rsqrt() * (A.sum(-1) > 0)
    S = (dinv[:, :, None] * A * dinv[:, None, :]).contiguous()
    iters = max(5, min(200, int(2e6 / (B * N))))
    for _ in range(3):
        y = gp.graph_filter(x, S, w, b, True, gp.NODE_MAJOR, gp.NODE_MAJOR)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        y = gp.graph_filter(x, S, w, b, True, gp.NODE_MAJOR, gp.NODE_MAJOR)
    e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / iters
    out.append({"B": B, "us": us, "agent_steps_per_s": B * N / us * 1e6,
                "alg_GBps": 4 * (128 + N + 128) * B * N / us * 1e-3})
print(json.dumps(out))
'''

if __name__ == "__main__":
    N = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    K = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(
        os.path.join(ROOT, "MEASURED_PEAKS.json")) else 3350.0     # H100 SXM data sheet, HBM3
    modes = [int(m) for m in sys.argv[3].split(",")] if len(sys.argv) > 3 else [1, 2, 3]
    for mode, name in ((1, "cuda-core"), (2, "wgmma-3xtf32"), (3, "wgmma-pair")):
        if mode not in modes:
            continue
        r = subprocess.run([sys.executable, "-c", CHILD % ROOT, str(N), str(K), str(mode)], capture_output=True, text=True)
        if r.returncode != 0:
            print(name, "FAILED", r.stderr[-400:])
            continue
        for row in json.loads(r.stdout.strip().splitlines()[-1]):
            print("%-12s N=%d K=%d B=%6d  %9.1f us  %8.2f M agent-steps/s  %7.1f GB/s algorithmic = %.3f of HBM peak (incl. tap prep launch)"
                  % (name, N, K, row["B"], row["us"], row["agent_steps_per_s"] / 1e6, row["alg_GBps"], row["alg_GBps"] / peak))
