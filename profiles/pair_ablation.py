"""Ablations of gf_fwd_pair_kernel ("pair_ablate" debug option): which producer stage bounds the tile time.
usage: python profiles/pair_ablation.py [B]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import gnn_pathplanning_b200 as gp
from gnn_pathplanning_b200 import _lib

B = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
N, K = 10, 3
torch.manual_seed(0)
w = ((torch.rand(128, 1, K, 128) - 0.5) * 0.2).cuda()
b = (torch.rand(128, 1) - 0.5).cuda()
x = torch.randn(B, N, 128, device="cuda")
S = torch.rand(B, N, N, device="cuda") * 0.2
_lib.set_debug_option("gf_mode", 3)
names = {0: "full kernel", 1: "no propagation", 2: "no operand stores", 3: "no propagation, no operand stores",
         4: "no x loads", 7: "producers only wait + arrive", 8: "no y stores", 15: "pipeline skeleton"}
for mask in (0, 1, 2, 3, 4, 7, 8, 15):
    _lib.set_debug_option("pair_ablate", mask)
    for _ in range(2):
        gp.graph_filter(x, S, w, b, True, gp.NODE_MAJOR, gp.NODE_MAJOR)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        gp.graph_filter(x, S, w, b, True, gp.NODE_MAJOR, gp.NODE_MAJOR)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / 5
    print("ablate %2d  %-36s %8.1f us   %.3f us per tile per CTA" % (mask, names[mask], us, us / (B / 12 / torch.cuda.get_device_properties(0).multi_processor_count)))
_lib.set_debug_option("pair_ablate", 0)
