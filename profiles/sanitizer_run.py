import sys
sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__))))
import numpy as np, torch
import gnn_pathplanning_b200 as gp
from gnn_pathplanning_b200 import synthetic
from oracle import planner_oracle as po
class Cfg:
    def __init__(self, n, k): self.num_agents, self.nGraphFilterTaps, self.device = n, k, torch.device("cuda")
def rel(a, b): return float(np.abs(a - b).max() / np.abs(b).max())
for (N, K, B, fe, gf) in [(10, 3, 70, "mma", "cuda"), (7, 2, 3, "mma", "cuda"), (10, 3, 450, "mma", "pair"), (10, 3, 8, "cuda", "cuda"),
                          (10, 3, 64, "mma", "auto"), (10, 2, 7, "cuda", "auto"), (10, 1, 1, "cuda", "auto")]:   # auto at N = 10: gf_small_mma_kernel
    sd = po.init_state_dict(K, seed=N); po.randomize_bn_stats(sd, seed=B)
    x, S = synthetic.make_batch(B, N, 20, seed=B)
    m = gp.DecentralPlannerNet(Cfg(N, K)); m.load_state_dict(sd); m = m.cuda().eval()
    m.set_feature_mode(fe); m.set_graph_filter_mode(gf)
    with torch.no_grad():
        m.addGSO(torch.from_numpy(S).cuda())
        got = torch.stack(m(torch.from_numpy(x).cuda())).cpu().numpy()
        ref = torch.stack(po.planner_forward(sd, torch.from_numpy(S), torch.from_numpy(x))).numpy()
    print(N, K, B, fe, gf, "rel err %.2e" % rel(got, ref), flush=True)
# rollout kernels
rng = np.random.default_rng(0)
cases = [synthetic.random_episode(rng, 10, 20, 0.1) for _ in range(5)]
ro = gp.BatchedRollout(10, 6.0).setup(np.stack([c[1] for c in cases]), np.stack([c[2] for c in cases]), np.stack([c[0] for c in cases]), 12)
sd = po.init_state_dict(3, seed=3); sd["actionsMLP.0.weight"] = sd["actionsMLP.0.weight"] * 40.0
m = gp.DecentralPlannerNet(Cfg(10, 3)); m.load_state_dict(sd); m = m.cuda().eval()
print("rollout steps", ro.run(m, poll_every=4), flush=True)
torch.cuda.synchronize()
print("done")
