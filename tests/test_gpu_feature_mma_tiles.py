"""GPU: the wgmma feature extractor (feature_mma_kernel) across the shapes of its work split -- partial 64-row blocks and
ragged 8-agent tiles, per-agent scales that differ by orders of magnitude inside one tile, and independence of an
episode's result from its position in the batch."""
import numpy as np
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-5


class Cfg:
    def __init__(self, n, k):
        self.num_agents, self.nGraphFilterTaps, self.device = n, k, torch.device("cuda")


def _mma_model(sd, N, K):
    import gnn_pathplanning_b200 as gp
    m = gp.DecentralPlannerNet(Cfg(N, K))
    m.load_state_dict(sd)
    m = m.cuda().eval()
    m.set_feature_mode("mma")
    return m


def _run(m, x, S):
    with torch.no_grad():
        m.addGSO(S.cuda())
        return torch.stack(m(x.cuda())).cpu().numpy()


@pytest.mark.parametrize("agents", list(range(1, 18)) + [63, 64, 65, 639, 640, 641, 10561])
def test_mma_agent_counts_vs_oracle(agents):
    """One agent per episode (N = 1), so the agent count is free: every tile fill and the partial last tile."""
    from gnn_pathplanning_b200 import synthetic
    from oracle import planner_oracle as po
    sd = po.init_state_dict(3, seed=agents)
    po.randomize_bn_stats(sd, seed=agents + 1)
    x, S = synthetic.make_batch(agents, 1, 20, seed=agents + 2)
    xt, St = torch.from_numpy(x), torch.from_numpy(S)
    with torch.no_grad():
        ref = torch.stack(po.planner_forward(sd, St, xt)).numpy()
    got = _run(_mma_model(sd, 1, 3), xt, St)
    assert rel_err(got, ref) <= TOL
    top2 = np.sort(ref, -1)
    clear = (top2[..., -1] - top2[..., -2]) > 1e-4 * np.abs(ref).max()
    assert np.array_equal(got.argmax(-1)[clear], ref.argmax(-1)[clear])


def test_mma_one_tile_magnitudes_2e_minus30_to_2e30():
    """One tile of 8 agents whose inputs span 2^-30 .. 2^30.  Biases, BatchNorm means and the GSO are zero, so the
    network is positively homogeneous and each agent's logits scale with its inputs: every agent is compared on its
    own, against a float64 oracle."""
    from oracle import planner_oracle as po
    N, K = 8, 3
    sd = po.init_state_dict(K, seed=11)
    po.randomize_bn_stats(sd, seed=12)
    for k in sd:
        if k.endswith("bias") or k.endswith("running_mean"):
            sd[k] = torch.zeros_like(sd[k])
    g = torch.Generator().manual_seed(13)
    scale = torch.pow(2.0, torch.linspace(-30, 30, N, dtype=torch.float64))
    x = (torch.rand(1, N, 3, 11, 11, generator=g, dtype=torch.float64) * scale.reshape(1, N, 1, 1, 1)).float()
    S = torch.zeros(1, N, N)
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    with torch.no_grad():
        ref = torch.stack(po.planner_forward(sd64, S.double(), x.double())).numpy()
    got = _run(_mma_model(sd, N, K), x, S)
    for a in range(N):
        assert np.abs(ref[a]).max() > 0, a
        assert rel_err(got[a], ref[a]) <= TOL, a


def test_mma_episode_permutation_is_bit_exact():
    """Permuting the episodes of a batch permutes the logits bit for bit: no row of a tile reads another row, and the
    per-agent scales depend on the agent alone (640 agents: the benchmark batch, 80 tiles)."""
    from gnn_pathplanning_b200 import synthetic
    from oracle import planner_oracle as po
    B, N, K = 64, 10, 3
    sd = po.init_state_dict(K, seed=21)
    po.randomize_bn_stats(sd, seed=22)
    x, S = synthetic.make_batch(B, N, 20, seed=23)
    xt, St = torch.from_numpy(x), torch.from_numpy(S)
    perm = torch.from_numpy(np.random.default_rng(24).permutation(B))
    m = _mma_model(sd, N, K)
    got = _run(m, xt, St)
    got_p = _run(m, xt[perm], St[perm])
    assert np.array_equal(got_p, got[:, perm.numpy()])
