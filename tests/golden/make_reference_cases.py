"""Generates tests/golden/reference_cases.npz: what tests/test_oracle_vs_reference.py and
tests/test_sim_oracle_vs_reference.py compare the oracle with, produced by the UNMODIFIED reference on CPU.

    GNNPP_REFERENCE_ROOT=<checkout of proroklab/gnn_pathplanning> python tests/golden/make_reference_cases.py

Inputs are rebuilt by the tests from the same seeds, so only the reference's outputs are stored.
"""
import contextlib
import hashlib
import io
import os
import sys
import warnings

import numpy as np
import torch

warnings.filterwarnings("ignore")
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import golden_io  # noqa: E402
from oracle import planner_oracle as po, ref_agent, ref_shim, ref_sim  # noqa: E402
import test_oracle_vs_reference as tov  # noqa: E402
import test_sim_oracle_vs_reference as tsv  # noqa: E402


def state_dict_digest(sd):
    """sha256 over the raw bytes of every tensor, in state_dict order."""
    h = hashlib.sha256()
    for k, v in sd.items():
        h.update(k.encode())
        h.update(v.detach().contiguous().numpy().tobytes())
    return h.hexdigest()


def main():
    assert ref_shim.available() and ref_agent.available(), "set GNNPP_REFERENCE_ROOT to a reference checkout"
    out = {}
    with contextlib.redirect_stdout(io.StringIO()):
        gml, dcp, _ = ref_shim.load()
    for K, N, B in tov.PLANNER_CASES:
        key = tov.case_key(K, N, B)
        torch.manual_seed(1337)
        m = dcp.DecentralPlannerNet(ref_shim.Config(N, K))
        out[key + "init_digest"] = np.array(state_dict_digest(m.state_dict()))
        sd = po.init_state_dict(K, seed=1337)
        po.randomize_bn_stats(sd)
        m.load_state_dict(sd)
        x, S = tov.planner_inputs(N, B)
        m.eval()
        m.addGSO(S.double())
        with torch.no_grad():
            out[key + "eval"] = torch.stack(m(x)).numpy()
        m.train()
        m.addGSO(S)
        out[key + "train"] = torch.stack(m(x)).detach().numpy()
        for k, v in m.state_dict().items():
            if "running" in k:
                out[key + "bn_" + k] = v.numpy()
    for i, (h, b, S, x) in enumerate(tov.filter_cases()):
        out["gf%d_y" % i] = gml.BatchLSIGF(h, S, x, b).numpy()
    for case in tsv.CASES:
        N, W, density, makespan, T, seed = case
        rng = np.random.default_rng(1000 + seed)
        c = ref_sim.make_case(rng, N, W, density, makespan)
        with ref_agent.reference_env(dropin=False) as agmod:
            ref = ref_sim.reference_rollout(agmod, c, T, seed, N)
        for k, v in ref.items():
            out[tsv.case_key(case) + k] = np.asarray(v)
    golden_io.savez_split(os.path.join(HERE, "reference_cases.npz"), out)


if __name__ == "__main__":
    main()
