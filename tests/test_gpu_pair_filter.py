"""GPU parity of the fp16-split pair graph filter (gf_fwd_pair_kernel: propagate in registers, 2-way fp16 split with
per-sample power-of-two scaling, wgmma with the taps streamed through a bulk-copy ring)
against the CPU oracle: standalone op through the C ABI, and inside the planner (fused ReLU + action MLP)."""
import numpy as np
import pytest
import torch

from conftest import rel_err

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]
TOL = 1e-5


@pytest.fixture()
def pair_mode():
    from gnn_pathplanning_b200 import _lib
    _lib.set_debug_option("gf_mode", 3)
    yield
    _lib.set_debug_option("gf_mode", 0)


def _case(B, N, K, seed, s_f64=False, rollout_like=True):
    gen = torch.Generator().manual_seed(seed)
    w = (torch.rand(128, 1, K, 128, generator=gen) - 0.5) * 0.2
    b = torch.rand(128, 1, generator=gen) - 0.5
    x = torch.randn(B, N, 128, generator=gen)
    if rollout_like:
        from gnn_pathplanning_b200 import synthetic
        S = np.stack([synthetic.gso_from_positions(np.random.default_rng(seed + i).integers(0, 14, size=(N, 2)), 6.0)
                      for i in range(B)])
        S = torch.from_numpy(S)
        S = S if s_f64 else S.float()
    else:
        S = (torch.rand(B, N, N, generator=gen) - 0.3) * 0.6         # dense, asymmetric, signed
        S = S.double() if s_f64 else S
    return w, b, x, S


def _oracle(w, b, x, S, relu):
    from oracle import planner_oracle as po
    y = po.batch_lsigf(w, S.unsqueeze(1), x.permute(0, 2, 1).contiguous(), b)      # [B,F,N]
    y = y.permute(0, 2, 1).contiguous()
    return torch.relu(y) if relu else y


@pytest.mark.parametrize("B,K,relu,bias,s_f64,rollout", [
    (1, 3, False, True, False, True), (5, 3, True, True, False, True), (12, 3, False, False, False, False),
    (13, 3, True, True, True, True), (24, 2, False, True, False, False), (25, 1, True, True, False, True),
    (300, 3, True, True, False, True), (4097, 3, False, True, False, True), (3553, 2, True, False, True, False),
])
def test_pair_kernel_vs_oracle(pair_mode, B, K, relu, bias, s_f64, rollout):
    import gnn_pathplanning_b200 as g
    N = 10
    w, b, x, S = _case(B, N, K, seed=B * 7 + K, s_f64=s_f64, rollout_like=rollout)
    ref = _oracle(w, b if bias else None, x, S, relu).numpy()
    y = g.graph_filter(x.cuda(), S.cuda(), w.cuda(), b.cuda() if bias else None, relu, g.NODE_MAJOR, g.NODE_MAJOR)
    torch.cuda.synchronize()
    err = rel_err(y.cpu().numpy(), ref)
    print("B=%d K=%d err %.2e" % (B, K, err))
    assert err <= TOL


def test_pair_kernel_dynamic_range_and_fp64_distance(pair_mode):
    """Per-sample scaling: samples whose signals differ by 12 orders of magnitude in one launch, each compared on its
    own scale; an all-zero sample; and the distance to a float64 evaluation next to the fp32 reference's own."""
    import gnn_pathplanning_b200 as g
    from oracle import planner_oracle as po
    N, K, B = 10, 3, 40
    w, b, x, S = _case(B, N, K, seed=77, rollout_like=False)
    mags = 10.0 ** torch.linspace(-6, 6, B)
    x = x * mags[:, None, None]
    x[7] = 0.0
    bz = torch.zeros_like(b)
    ref = _oracle(w, bz, x, S, False).numpy()
    y = g.graph_filter(x.cuda(), S.cuda(), w.cuda(), bz.cuda(), False, g.NODE_MAJOR, g.NODE_MAJOR).cpu().numpy()
    for i in range(B):
        if i == 7:
            assert np.all(y[i] == 0.0)
        else:
            assert rel_err(y[i], ref[i]) <= TOL, (i, float(mags[i]))
    y64 = po.graph_filter_f64(w.numpy(), bz.numpy(), S.numpy(), x.permute(0, 2, 1).numpy()).transpose(0, 2, 1)
    worst_cuda = max(rel_err(y[i], y64[i]) for i in range(B) if i != 7)
    worst_ref = max(rel_err(ref[i], y64[i]) for i in range(B) if i != 7)
    print("distance to float64: pair kernel %.2e, fp32 reference %.2e" % (worst_cuda, worst_ref))
    assert worst_cuda <= TOL


def test_pair_kernel_large_gso_entries(pair_mode):
    """A GSO that is NOT a normalised adjacency (entries up to 3, column sums ~15): the scale bound follows the
    largest absolute column sum, so nothing overflows fp16."""
    import gnn_pathplanning_b200 as g
    N, K, B = 10, 3, 30
    w, b, x, S = _case(B, N, K, seed=5, rollout_like=False)
    S = S * 5.0
    ref = _oracle(w, b, x, S, True).numpy()
    y = g.graph_filter(x.cuda(), S.cuda(), w.cuda(), b.cuda(), True, g.NODE_MAJOR, g.NODE_MAJOR).cpu().numpy()
    assert np.isfinite(y).all() and rel_err(y, ref) <= TOL


class Cfg:
    def __init__(self, n, k):
        self.num_agents, self.nGraphFilterTaps, self.device = n, k, torch.device("cuda")


@pytest.mark.parametrize("K,B", [(3, 64), (3, 1000), (2, 37), (3, 1)])
def test_planner_with_pair_filter(K, B):
    import gnn_pathplanning_b200 as gp
    from gnn_pathplanning_b200 import synthetic
    from oracle import planner_oracle as po
    N = 10
    sd = po.init_state_dict(K, seed=B + K)
    po.randomize_bn_stats(sd, seed=B)
    m = gp.DecentralPlannerNet(Cfg(N, K))
    m.load_state_dict(sd)
    m = m.cuda().eval()
    m.set_graph_filter_mode("pair")
    x, S = synthetic.make_batch(B, N, 20, seed=B + 3)
    xt, St = torch.from_numpy(x), torch.from_numpy(S)
    with torch.no_grad():
        ref = torch.stack(po.planner_forward(sd, St, xt)).numpy()
        m.addGSO(St.cuda())
        got = torch.stack(m(xt.cuda())).cpu().numpy()
        m.addGSO(St.double().cuda())                      # float64 GSO, as the rollout simulator hands over
        got64 = torch.stack(m(xt.cuda())).cpu().numpy()
    assert rel_err(got, ref) <= TOL and rel_err(got64, ref) <= TOL
    top2 = np.sort(ref, -1)
    clear = (top2[..., -1] - top2[..., -2]) > 1e-4 * np.abs(ref).max()
    assert np.array_equal(got.argmax(-1)[clear], ref.argmax(-1)[clear])


def test_pair_mode_outside_envelope_is_loud(pair_mode):
    import gnn_pathplanning_b200 as g
    w, b, x, S = _case(4, 10, 3, seed=1)
    with pytest.raises(NotImplementedError):
        g.graph_filter(torch.randn(4, 20, 128).cuda(), torch.rand(4, 20, 20).cuda(), w.cuda(), b.cuda(), False,
                       g.NODE_MAJOR, g.NODE_MAJOR)
