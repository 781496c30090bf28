"""CPU: host-side logic -- the C-ABI library loads and exports every declared symbol, the
drop-in modules keep the reference's API surface, the product never imports the oracle."""
import os
import re

import numpy as np
import pytest
import torch

from conftest import ROOT, rel_err


class Cfg:
    def __init__(self, n, k):
        self.num_agents, self.nGraphFilterTaps, self.device = n, k, "cpu"


def test_library_exports_every_declared_symbol():
    from gnn_pathplanning_b200 import _lib
    lib = _lib.load()           # loads without a GPU (no compute calls here)
    for fname, listed in (("gnnpp_b200.h", _lib.EXPORTED), ("gnnpp_b200_debug.h", _lib.DEBUG_EXPORTED)):
        header = open(os.path.join(ROOT, "include", fname)).read()
        declared = sorted(set(re.findall(r"\b(gpp_[a-z_0-9]+)\s*\(", header)))
        assert declared, "no declarations parsed"
        for name in declared:
            assert hasattr(lib, name), name
        assert sorted(listed) == declared, fname
    # the drop-in boundary carries no debug / test hooks
    assert not [n for n in _lib.EXPORTED if "debug" in n]
    assert lib.gpp_abi_version() == 1


def test_state_dict_surface_and_init_match_reference(golden):
    import gnn_pathplanning_b200 as gp
    for f, K in (("planner_K3.npz", 3), ("planner_K2.npz", 2)):
        g = golden(f)
        torch.manual_seed(1337)
        m = gp.DecentralPlannerNet(Cfg(10, K))
        sd = m.state_dict()
        keys = sorted(sd.keys())
        assert keys == [str(k) for k in g["init_keys"]]
        for k in keys:
            assert tuple(sd[k].shape) == tuple(g["sd_" + k].shape), k
        fp = np.array([float(sd[k].double().sum()) for k in keys])
        assert np.allclose(fp, g["init_fingerprint"], rtol=0, atol=1e-9)     # same init as the reference
        assert (m.numAgents, m.numFeatures2Share, m.L, m.F, m.K, m.E, m.bias) == (10, 128, 1, [128, 128], [K], 1, True)
        names = [n for n, _ in m.named_parameters()]
        assert any(n.startswith("GFL.") for n in names) and any(n.startswith("actionsMLP.") for n in names)


def test_graph_filter_module_surface():
    import gnn_pathplanning_b200 as gp
    lay = gp.GraphFilterBatch(6, 10, 3)
    assert tuple(lay.weight.shape) == (10, 1, 3, 6) and tuple(lay.bias.shape) == (10, 1)
    bound = 1.0 / np.sqrt(6 * 3)
    assert float(lay.weight.detach().abs().max()) <= bound and float(lay.bias.detach().abs().max()) <= bound
    assert gp.GraphFilterBatch(6, 10, 3, bias=False).bias is None
    assert "no GSO stored" in lay.extra_repr()
    with pytest.raises(AssertionError):
        lay.addGSO(torch.rand(2, 5, 5))
    lay.addGSO(torch.rand(2, 1, 5, 5))
    assert "GSO stored" in lay.extra_repr() and lay.N == 5
    with pytest.raises(RuntimeError, match="does not fall back"):
        lay(torch.rand(2, 6, 5))                         # CPU tensors: loud failure, no fallback
    with pytest.raises(NotImplementedError):                 # E != 1 is outside the planner path
        gp.graph_filter(torch.rand(1, 6, 5), torch.rand(1, 2, 5, 5), torch.rand(10, 2, 3, 6))


def test_planner_api_asserts_on_cpu():
    import gnn_pathplanning_b200 as gp
    m = gp.DecentralPlannerNet(Cfg(4, 2))
    with pytest.raises(AssertionError):
        m.addGSO(torch.rand(2, 1, 4, 4))
    m.addGSO(torch.rand(2, 4, 4))
    assert tuple(m.S.shape) == (2, 1, 4, 4)
    with pytest.raises(RuntimeError, match="does not fall back"):
        m(torch.rand(2, 4, 3, 11, 11))


def test_dropin_hook_routes_three_names_and_nothing_else(tmp_path):
    """install_dropin() on a stand-in tree laid out like the reference (package __init__s that eagerly import
    every sibling module, as gnn_pathplanning/utils/__init__.py:6-10 does): the three hot-path module names
    resolve to this package, every other module of the same packages still comes from the tree."""
    import gnn_pathplanning_b200 as gp
    import sys
    eager = ("import os, sys\npath = os.path.dirname(os.path.abspath(__file__))\n"
             "for py in [f[:-3] for f in os.listdir(path) if f.endswith('.py') and f != '__init__.py']:\n"
             "    __import__('.'.join([__name__, py]), fromlist=[py])\n")
    tree = {"graphs/__init__.py": eager, "graphs/weights_initializer.py": "ORIGIN = 'tree'\n",
            "graphs/models/__init__.py": eager, "graphs/models/decentralplanner.py": "ORIGIN = 'tree'\n",
            "graphs/losses/__init__.py": eager, "graphs/losses/cross_entropy.py": "ORIGIN = 'tree'\n",
            "utils/__init__.py": eager, "utils/metrics.py": "ORIGIN = 'tree'\n",
            "utils/graphUtils/__init__.py": "", "utils/graphUtils/graphML.py": "ORIGIN = 'tree'\n",
            "utils/graphUtils/graphTools.py": "ORIGIN = 'tree'\n"}
    for rel, src in tree.items():
        f = tmp_path / rel
        f.parent.mkdir(parents=True, exist_ok=True)
        f.write_text(src)
    saved = {k: v for k, v in sys.modules.items() if k.split(".")[0] in ("graphs", "utils")}
    for k in saved:
        del sys.modules[k]
    sys.path.insert(0, str(tmp_path))
    try:
        gp.install_dropin()
        from graphs.models.decentralplanner import DecentralPlannerNet
        from graphs.weights_initializer import weights_init
        import utils.graphUtils.graphML as gml
        assert DecentralPlannerNet is gp.DecentralPlannerNet
        assert gml.GraphFilterBatch is gp.GraphFilterBatch and gml.BatchLSIGF is gp.BatchLSIGF
        assert weights_init is gp.weights_init
        import graphs.losses.cross_entropy as ce
        import utils.metrics as metrics
        import utils.graphUtils.graphTools as gt
        assert ce.ORIGIN == metrics.ORIGIN == gt.ORIGIN == "tree"
        import graphs
        assert graphs.weights_initializer.weights_init is gp.weights_init      # the eager __init__ got the override too
    finally:
        from gnn_pathplanning_b200 import dropin
        dropin.uninstall()
        sys.path.remove(str(tmp_path))
        for k in [k for k in sys.modules if k.split(".")[0] in ("graphs", "utils")]:
            del sys.modules[k]
        sys.modules.update(saved)


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "gnn_pathplanning_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, re.M), f
                assert "planner_oracle" not in src and "ref_shim" not in src, f


def test_bench_reference_arm_prints_the_contract_line():
    """`bench.py --impl reference` (the CPU arm the driver times beside the GPU arm) runs without a GPU and prints ONE JSON
    line with the contract's keys; its `config` is the same dict the GPU arm prints."""
    import json
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1"],
                       capture_output=True, text=True, timeout=600, cwd=root)
    assert r.returncode == 0, r.stderr[-500:]
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "agent-steps/s" and d["higher_is_better"] is True
    for k in ("metric", "value", "n_gpus", "steps", "warmup", "ms_per_step", "scaling", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0 and d["e2e"]["value"] == d["value"]
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1
    sys.path.insert(0, root)
    import bench
    assert d["config"] == bench.config_dict(1)
