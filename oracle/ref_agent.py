"""TEST INFRASTRUCTURE ONLY -- run the reference's own AGENT code (agents/decentralplannerlocal.py,
utils/multirobotsim_dcenlocal.py, utils/metrics.py, graphs/losses/*) from the reference checkout, unmodified,
either against the reference's own model or against this repo's drop-in modules.

Needs a reference checkout (GNNPP_REFERENCE_ROOT); only the golden-data generators use it.  Used by
  * tests/golden/make_agent_trace.py   reference agent + reference model  -> tests/golden/agent_trace.npz
  * tests/test_reference_agent_dropin.py   reference agent + gnn_pathplanning_b200.install_dropin()

The reference's package __init__s import every sibling module eagerly, which pulls in plotting /
logging packages that are absent here (matplotlib, seaborn, tensorboardX, easydict, torchsummaryX,
hashids, skimage, drawSvg, plotly): they are stubbed -- none of them is on the path under test.
"""
from __future__ import annotations

import contextlib
import importlib
import importlib.abc
import importlib.util
import io
import logging
import os
import random
import sys
import types

import numpy as np
import torch

REF_ROOT = os.environ.get("GNNPP_REFERENCE_ROOT", "")
STUBBED = ("matplotlib", "seaborn", "tensorboardX", "easydict", "torchsummaryX", "hashids", "skimage", "drawSvg",
           "plotly", "mpl_toolkits")
REF_PACKAGES = ("agents", "utils", "graphs", "dataloader", "onlineExpert", "offlineExpert")


def available() -> bool:
    return os.path.isfile(os.path.join(REF_ROOT, "agents", "decentralplannerlocal.py"))


class EasyDict(dict):
    """Minimal attribute dict (the reference's config type, utils/config.py)."""

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)

    def __setattr__(self, k, v):
        self[k] = v


class _Anything:
    """Callable / subclassable placeholder for plotting classes never touched on the path."""

    def __init__(self, *a, **k):
        pass

    def __call__(self, *a, **k):
        return _Anything()

    def __getattr__(self, k):
        return _Anything()

    def __getitem__(self, k):
        return _Anything()

    def __setitem__(self, k, v):
        pass

    def __iter__(self):
        return iter(())

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


class _StubModule(types.ModuleType):
    def __getattr__(self, k):
        if k.startswith("__"):
            raise AttributeError(k)
        if self.__name__ == "easydict" and k == "EasyDict":
            return EasyDict
        if k[:1].isupper():
            return type(k, (_Anything,), {})          # classes: may be subclassed at import time
        return _Anything()                            # functions / objects (plt.rcParams[...] = ...)


class _StubLoader(importlib.abc.Loader):
    def create_module(self, spec):
        m = _StubModule(spec.name)
        m.__path__ = []
        return m

    def exec_module(self, module):
        return None


class _StubFinder(importlib.abc.MetaPathFinder):
    def find_spec(self, fullname, path=None, target=None):
        if fullname.split(".")[0] in STUBBED:
            try:                                        # never hide a real installation
                for f in sys.meta_path:
                    if f is self or not hasattr(f, "find_spec"):
                        continue
                    s = f.find_spec(fullname, path, target)
                    if s is not None:
                        return s
            except Exception:
                pass
            return importlib.util.spec_from_loader(fullname, _StubLoader(), is_package=True)
        return None


def _purge():
    for k in [k for k in sys.modules if k.split(".")[0] in REF_PACKAGES or k.split(".")[0] in STUBBED]:
        if isinstance(sys.modules[k], _StubModule) or k.split(".")[0] in REF_PACKAGES:
            del sys.modules[k]


@contextlib.contextmanager
def reference_env(dropin: bool):
    """sys.path / sys.modules set up so that `import agents.decentralplannerlocal` runs the reference's
    agent module; `dropin` = route the three hot-path module names to gnn_pathplanning_b200."""
    assert available(), "reference tree not present at %s" % REF_ROOT
    saved_mods = {k: v for k, v in sys.modules.items() if k.split(".")[0] in REF_PACKAGES}
    _purge()
    finder = _StubFinder()
    sys.meta_path.append(finder)
    sys.path.insert(0, REF_ROOT)
    cwd = os.getcwd()
    if dropin:
        import gnn_pathplanning_b200 as gp
        gp.install_dropin()
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            agmod = importlib.import_module("agents.decentralplannerlocal")
        yield agmod
    finally:
        os.chdir(cwd)
        if dropin:
            from gnn_pathplanning_b200 import dropin as _d
            _d.uninstall()
        sys.meta_path.remove(finder)
        sys.path.remove(REF_ROOT)
        _purge()
        sys.modules.update(saved_mods)


def make_config(num_agents=10, K=3, device="cpu", rate_maxstep=2):
    c = EasyDict()
    c.num_agents, c.nGraphFilterTaps, c.device = num_agents, K, torch.device(device)
    c.rate_maxstep, c.commR, c.mode, c.log_anime = rate_maxstep, 6, "train", False
    c.exp_name, c.log_interval, c.learning_rate, c.weight_decay = "dropin-test", 1000, 1e-3, 1e-5
    return c


class _Writer:
    def __init__(self):
        self.scalars = []

    def add_scalar(self, tag, v, it):
        self.scalars.append((tag, float(v), int(it)))


class _Loader(list):
    dataset = [0]


def make_agent(agmod, model, config, train_batches):
    """A DecentralPlannerAgentLocal whose __init__ (dataset paths, checkpoint dirs, TensorBoard) is
    bypassed: exactly the attributes train_one_epoch (:276-326) and mutliAgent_ActionPolicy (:535-648)
    read are filled in, with the reference's own simulator / recorder / loss classes."""
    cls = agmod.DecentralPlannerAgentLocal
    ag = object.__new__(cls)
    ag.config = config
    ag.logger = logging.getLogger("ref-agent")
    ag.model = model
    ag.loss = agmod.CrossEntropyLoss()
    ag.optimizer = torch.optim.Adam(model.parameters(), lr=config.learning_rate, weight_decay=config.weight_decay)
    ag.current_epoch, ag.current_iteration = 0, 0
    ag.summary_writer = _Writer()
    dl = types.SimpleNamespace()
    dl.train_loader = _Loader(train_batches)
    ag.data_loader = dl
    with contextlib.redirect_stdout(io.StringIO()):
        ag.robot = agmod.multiRobotSim(config)
    ag.recorder = agmod.MonitoringMultiAgentPerformance(config)
    return ag


def make_case(num_agents, map_w, seed, horizon=12):
    """One rollout case in the test-loader format of Dataloader_dcplocal_notTF_onlineExpert.py:184-205:
    input [1,2,N,2] (goal, start positions), target [1,N,T,5] one-hot expert actions (all 'stop' here:
    only used for the target-path metrics), makespan [1], map [1,W,W]."""
    from gnn_pathplanning_b200 import synthetic
    rng = np.random.default_rng(seed)
    m, starts, goals = synthetic.random_episode(rng, num_agents, map_w)
    inp = torch.from_numpy(np.stack([goals, starts])[None].astype(np.float32))
    tgt = torch.zeros(1, num_agents, horizon, 5)
    tgt[..., 4] = 1.0
    return inp, tgt, torch.tensor([float(horizon)]), torch.from_numpy(m[None].astype(np.float32))


class Recorder(torch.nn.Module):
    """Wraps a planner module and records what the agent hands it / gets back each call."""

    def __init__(self, inner):
        super().__init__()
        self.inner = inner
        self.calls = []
        self._S = None

    def addGSO(self, S):
        self._S = S
        self.inner.addGSO(S)

    def forward(self, x):
        out = self.inner(x)
        self.calls.append((x.detach().cpu().clone(), self._S.detach().cpu().clone(),
                           torch.stack([o.detach().cpu() for o in out])))
        return out


def run_agent_trace(agmod, model, config, batch, case):
    """One train_one_epoch batch, then one rollout case, through the reference's agent methods.
    Returns dict of numpy arrays (the golden trace)."""
    rec = Recorder(model)
    ag = make_agent(agmod, rec, config, [batch])
    ag.model = rec
    ag.optimizer = torch.optim.Adam(model.parameters(), lr=config.learning_rate, weight_decay=config.weight_decay)
    ag.train_one_epoch()
    out = {"train_loss": np.float64(ag.summary_writer.scalars[-1][1]),
           "train_logits": rec.calls[0][2].numpy()}
    rec.calls.clear()
    # the rollout below runs on the parameters / BatchNorm statistics this one optimizer step produced
    out.update({"after_" + k: v.detach().cpu().numpy().copy() for k, v in model.state_dict().items()})
    model.eval()
    random.seed(1337)
    with torch.no_grad():
        res = ag.mutliAgent_ActionPolicy(case[0].to(config.device), case[1].to(config.device), case[2], case[3], 0)
    out["rollout_x"] = np.stack([c[0].numpy() for c in rec.calls])          # [T,1,N,3,11,11]
    out["rollout_S"] = np.stack([c[1].numpy() for c in rec.calls])          # [T,1,N,N] float64
    out["rollout_logits"] = np.stack([c[2].numpy() for c in rec.calls])     # [T,N,1,5]
    N = config.num_agents
    paths = [ag.robot.status_MultiAgent["agent%d" % i]["path_predict"] for i in range(N)]
    T = len(rec.calls)
    out["rollout_pos"] = np.array([[[float(paths[i][t][0][0]), float(paths[i][t][0][1])] for i in range(N)]
                                   for t in range(T + 1) if all(t in p for p in paths)])
    out["rollout_actions"] = np.array([[int(a) for a in ag.robot.status_MultiAgent["agent%d" % i]["action_predict"]]
                                       for i in range(N)])
    out["all_reach_goal"] = np.int64(bool(res[0]))
    return out
