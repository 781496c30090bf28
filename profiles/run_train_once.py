import os, sys
sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__))))
import torch
import gnn_pathplanning_b200 as gp
from gnn_pathplanning_b200 import synthetic
from oracle import planner_oracle as po
class Cfg:
    num_agents, nGraphFilterTaps, device = 10, 3, torch.device("cuda")
sd = po.init_state_dict(3, seed=1)
x, S = synthetic.make_batch(64, 10, 20, seed=3)
tt = torch.from_numpy(synthetic.random_targets(64, 10, seed=4)).cuda()
xt, St = torch.from_numpy(x).cuda(), torch.from_numpy(S).cuda()
m = gp.DecentralPlannerNet(Cfg()); m.load_state_dict(sd); m = m.cuda().train()
for _ in range(3):
    m.zero_grad(); m.addGSO(St); loss = gp.planner_loss(m.forward_logits(xt), tt); loss.backward()
torch.cuda.synchronize()
