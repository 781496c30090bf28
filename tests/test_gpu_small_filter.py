"""GPU parity of the small-batch wgmma graph filter (gf_small_mma_kernel: N = 10, K <= 3, below 4,096 node rows --
the filter of the benchmark configuration and of rollout steps) through the planner's C ABI: against the CPU oracle
and against the CUDA-core kernel of the same library, at ragged tile counts, float64 GSOs, signed / badly scaled
GSOs (per-sample power-of-two scaling), isolated agents and the largest batch the kernel takes.
Reference: gnn_pathplanning/utils/graphUtils/graphML.py:2342-2366, graphs/models/decentralplanner.py:284-318."""
import numpy as np
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-5


class Cfg:
    def __init__(self, n, k):
        self.num_agents, self.nGraphFilterTaps, self.device = n, k, torch.device("cuda")


def _model(sd, K):
    import gnn_pathplanning_b200 as gp
    m = gp.DecentralPlannerNet(Cfg(10, K))
    m.load_state_dict(sd)
    return m.cuda().eval()


def _run(m, x, S, mode):
    m.set_graph_filter_mode(mode)
    m.addGSO(S.cuda())
    with torch.no_grad():
        return torch.stack(m(x.cuda())).cpu().numpy()


@pytest.mark.parametrize("K", [1, 2, 3])
@pytest.mark.parametrize("B", [1, 5, 6, 7, 13, 64, 409])       # 409 x 10 = 4,090 rows: the last size below the pair kernel
def test_vs_oracle_and_cuda_core_kernel(K, B):
    from gnn_pathplanning_b200 import synthetic
    from oracle import planner_oracle as po
    sd = po.init_state_dict(K, seed=40 + K)
    po.randomize_bn_stats(sd, seed=B)
    m = _model(sd, K)
    x, S = synthetic.make_batch(B, 10, 20, seed=3 * B + K)
    xt, St = torch.from_numpy(x), torch.from_numpy(S)
    with torch.no_grad():
        ref = torch.stack(po.planner_forward(sd, St, xt)).numpy()
    got = _run(m, xt, St, "auto")
    assert rel_err(got, ref) <= TOL
    assert rel_err(got, _run(m, xt, St, "cuda")) <= TOL
    top2 = np.sort(ref, -1)
    clear = (top2[..., -1] - top2[..., -2]) > 1e-4 * np.abs(ref).max()
    assert np.array_equal(got.argmax(-1)[clear], ref.argmax(-1)[clear])


@pytest.mark.parametrize("case", ["f64", "signed_large", "tiny", "isolated", "mixed_scales"])
def test_gso_edge_cases(case):
    """The kernel scales every sample by a power of two from max|x| * max(1, max column sum |S|)^(K-1) before the fp16
    split; these GSOs move that bound over ~40 binades inside one batch."""
    from gnn_pathplanning_b200 import synthetic
    from oracle import planner_oracle as po
    K, B = 3, 20
    sd = po.init_state_dict(K, seed=77)
    po.randomize_bn_stats(sd, seed=78)
    m = _model(sd, K)
    x, S = synthetic.make_batch(B, 10, 20, seed=91)
    rng = np.random.default_rng(5)
    if case == "f64":
        S = S.astype(np.float64)                         # the rollout passes float64 GSOs (S.float() in BatchLSIGF)
    elif case == "signed_large":
        S = (S * rng.choice([-1.0, 1.0], size=S.shape) * 37.0).astype(np.float32)
    elif case == "tiny":
        S = (S * 1e-6).astype(np.float32)
    elif case == "isolated":
        S[::2] = 0.0                                     # no neighbours at all: z_1 = z_2 = 0
    elif case == "mixed_scales":
        S = (S * (10.0 ** rng.uniform(-6, 3, size=(B, 1, 1)))).astype(np.float32)
    xt, St = torch.from_numpy(x), torch.from_numpy(S)
    with torch.no_grad():
        ref = torch.stack(po.planner_forward(sd, St, xt)).numpy()
    got = _run(m, xt, St, "auto")
    assert np.isfinite(got).all()
    assert rel_err(got, ref) <= TOL
    assert rel_err(got, _run(m, xt, St, "cuda")) <= TOL


def test_host_buffer_entry_points_use_the_same_kernel():
    """infer_host (zero-copy pinned buffers) and infer_host_async / wait at the benchmark size."""
    from gnn_pathplanning_b200 import synthetic
    from oracle import planner_oracle as po
    K, B = 3, 64
    sd = po.init_state_dict(K, seed=11)
    po.randomize_bn_stats(sd, seed=12)
    m = _model(sd, K)
    x, S = synthetic.make_batch(B, 10, 20, seed=13)
    xt, St = torch.from_numpy(x).pin_memory(), torch.from_numpy(S).pin_memory()
    with torch.no_grad():
        ref = torch.stack(po.planner_forward(sd, St, xt)).numpy()
    assert rel_err(m.infer_host(xt, St).numpy(), ref) <= TOL
    outs = [torch.empty(10, B, 5).pin_memory() for _ in range(3)]
    tickets = [m.infer_host_async(xt, St, o) for o in outs]
    for t, o in zip(tickets, outs):
        m.wait(t)
        assert rel_err(o.numpy(), ref) <= TOL


def test_device_async_pipeline_matches_oracle_and_sequential_calls():
    """infer_async / join (gpp_planner_forward_async): independent batches of different sizes in flight over the library's
    compute lanes, device tensors in and out, interleaved with ordinary forward calls on the same module."""
    from gnn_pathplanning_b200 import synthetic
    from oracle import planner_oracle as po
    K = 3
    sd = po.init_state_dict(K, seed=21)
    po.randomize_bn_stats(sd, seed=22)
    m = _model(sd, K)
    m.set_graph_filter_mode("auto")
    sizes = [64, 7, 64, 450, 1, 64, 13, 64, 64, 30, 64, 64]          # 450 x 10 rows: the CTA-pair filter kernel
    batches, refs = [], []
    for i, B in enumerate(sizes):
        x, S = synthetic.make_batch(B, 10, 20, seed=500 + i)
        if i % 3 == 1:
            S = S.astype(np.float64)
        xt, St = torch.from_numpy(x), torch.from_numpy(S)
        with torch.no_grad():
            refs.append(torch.stack(po.planner_forward(sd, St, xt)).numpy())
        batches.append((xt.cuda(), St.cuda()))
    torch.cuda.synchronize()
    inflight, outs = [], [None] * len(sizes)
    with torch.no_grad():
        for i, (xd, Sd) in enumerate(batches):
            tk, out = m.infer_async(xd, Sd)
            inflight.append((tk, i, out))
            if i == 5:                                   # a plain call in the middle of the pipeline
                m.addGSO(batches[0][1])
                mid = torch.stack(m(batches[0][0])).cpu().numpy()
                assert rel_err(mid, refs[0]) <= TOL
            if len(inflight) >= 6:
                tk0, j, o = inflight.pop(0)
                m.join(tk0)                              # device-side wait on the current stream
                outs[j] = o.clone()
        for tk0, j, o in inflight:
            m.wait(tk0)                                  # host-side wait
            outs[j] = o.clone()
    torch.cuda.synchronize()
    for j, B in enumerate(sizes):
        assert rel_err(outs[j].cpu().numpy(), refs[j]) <= TOL, (j, B)
