"""A few planner forwards (for ncu captures).  usage: run_planner_once.py [B N gf_mode fe_mode]"""
import sys
sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__))))
import torch
import gnn_pathplanning_b200 as gp
from gnn_pathplanning_b200 import synthetic

class Cfg:
    def __init__(self, n, k):
        self.num_agents, self.nGraphFilterTaps, self.device = n, k, torch.device("cuda")

B = int(sys.argv[1]) if len(sys.argv) > 1 else 64
N = int(sys.argv[2]) if len(sys.argv) > 2 else 10
m = gp.DecentralPlannerNet(Cfg(N, 3)).cuda().eval()
m.set_graph_filter_mode(sys.argv[3] if len(sys.argv) > 3 else "auto"); m.set_feature_mode(sys.argv[4] if len(sys.argv) > 4 else "auto")
x, S = synthetic.make_batch(B, N, 20, seed=1)
xt, St = torch.from_numpy(x).cuda(), torch.from_numpy(S).cuda()
m.addGSO(St)
with torch.no_grad():
    for _ in range(6):
        out = m(xt)
torch.cuda.synchronize()
print("ok", float(out[0].sum()))
