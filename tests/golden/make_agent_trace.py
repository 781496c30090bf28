"""Generates tests/golden/agent_trace.npz by running the reference's own AGENT code
(agents/decentralplannerlocal.py: train_one_epoch :276-326 on one batch, then one rollout case through
mutliAgent_ActionPolicy :535-648 with the real simulator) against the reference's own model on CPU.

Run with a reference checkout:   GNNPP_REFERENCE_ROOT=<checkout> python tests/golden/make_agent_trace.py
Consumed by tests/test_gpu_agent_trace.py (GPU: the recorded calls replayed on the CUDA module).
"""
import os
import sys
import warnings

import numpy as np
import torch

warnings.filterwarnings("ignore")
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import golden_io  # noqa: E402
from oracle import ref_agent  # noqa: E402
from oracle import planner_oracle as po  # noqa: E402
from gnn_pathplanning_b200 import synthetic  # noqa: E402

N, K, B, MAP_W = 10, 3, 16, 20


def inputs():
    sd = po.init_state_dict(K, seed=1337)
    po.randomize_bn_stats(sd)
    # a freshly initialised policy answers "stop" everywhere; a larger action head makes the argmax depend on
    # the features, so the rollout really moves agents (edge / obstacle / inter-robot shielding all fire)
    sd["actionsMLP.0.weight"] = sd["actionsMLP.0.weight"] * 40.0
    sd["GFL.0.weight"] = sd["GFL.0.weight"] * 3.0
    x, S = synthetic.make_batch(B, N, MAP_W, seed=77)
    tgt = synthetic.random_targets(B, N, seed=78)
    # train-loader item format (Dataloader_dcplocal_notTF_onlineExpert.py:142-157): input, target, step, GSO, map
    batch = (torch.from_numpy(x), torch.from_numpy(tgt), torch.zeros(B), torch.from_numpy(S), torch.zeros(B, 1))
    case = ref_agent.make_case(N, MAP_W, seed=79)
    return sd, batch, case


def main():
    sd, batch, case = inputs()
    cfg = ref_agent.make_config(N, K, "cpu")
    with ref_agent.reference_env(dropin=False) as agmod:
        torch.manual_seed(1337)
        model = agmod.DecentralPlannerNet(cfg)
        assert model.__class__.__module__ == "graphs.models.decentralplanner"
        model.load_state_dict(sd)
        tr = ref_agent.run_agent_trace(agmod, model, cfg, batch, case)
    out = {"N": np.int64(N), "K": np.int64(K), "B": np.int64(B)}
    out.update({"sd_" + k: v.numpy() for k, v in sd.items()})
    out.update({"batch_x": batch[0].numpy(), "batch_target": batch[1].numpy(), "batch_S": batch[3].numpy(),
                "case_input": case[0].numpy(), "case_target": case[1].numpy(), "case_makespan": case[2].numpy(),
                "case_map": case[3].numpy()})
    out.update(tr)
    path = os.path.join(HERE, "agent_trace.npz")
    golden_io.savez_split(path, dict(out))
    print("wrote", path, "rollout steps:", tr["rollout_x"].shape[0], "train loss %.6f" % tr["train_loss"],
          "all_reach_goal", int(tr["all_reach_goal"]))


if __name__ == "__main__":
    main()
