"""The fused update chain (ops.update_chain, k_update_chain) against the five tensor-core launches it replaces in the RAFT loop
(corr-motion head, MotionEncoder.conv, ConvGRU [z|r] and q, flow-head fc1 pre-transform): the results must be the same bits,
since the fused kernel runs the same k-block order, 3xTF32 split, wgmma shapes and epilogue formulas on the same fp32 values.

  * the kernel alone at the bench batch and at a batch with more tiles than SMs (a CTA crosses tiles and samples), with
    random and trained-like weights (negative and > 1 PReLU slopes, negative GroupNorm gammas); outputs NaN-prefilled
  * whole forwards, fused loop against the unfused one (ops.fuse_update_chain = False): RSF and RSF_refine, fp32 and bf16 state
  * CUDA-graph replay against eager under torch.use_deterministic_algorithms(True)
  * four launches fewer per iteration
"""
import types

import pytest
import torch

from conftest import default_weights

pytestmark = pytest.mark.gpu

LEVELS, SCALE = 3, 0.25


@pytest.fixture(scope='module')
def dev():
    return torch.device('cuda:0')


@pytest.fixture
def unfused():
    from pvraft_b200 import ops

    class Switch:
        def __enter__(self):
            ops.fuse_update_chain = False

        def __exit__(self, *exc):
            ops.fuse_update_chain = True
    yield Switch()
    ops.fuse_update_chain = True


def make_model(dev, k=128, refine=False, seed=0):
    from pvraft_b200 import RSF, RSF_refine
    args = types.SimpleNamespace(corr_levels=LEVELS, base_scales=SCALE, truncate_k=k)
    m = (RSF_refine if refine else RSF)(args)
    m.load_state_dict(default_weights(refine=refine, seed=seed, args=args), strict=True)
    return m.to(dev).eval()


def clouds(b, n, seed, dev):
    g = torch.Generator().manual_seed(seed)
    pc1 = 10.0 * torch.rand(b, n, 3, generator=g)
    pc2 = pc1 + 0.1 * torch.randn(b, n, 3, generator=g)
    return pc1.to(dev), pc2.to(dev)


def chain_inputs(model, b, n, dev, seed, regime):
    """Random per-point operands of the chain and a GroupNorm-sum table of y1 consistent with it."""
    g = torch.Generator().manual_seed(seed)
    cb, ub = model.corr_block, model.update_block
    with torch.no_grad():
        if regime == 'trained':   # negative and > 1 PReLU slopes, negative GroupNorm gammas
            cb.out_conv[2].weight.fill_(-0.7)
            cb.out_conv[1].weight.copy_(torch.randn(128, generator=g).to(dev) * 1.5)
            for conv in (ub.gru.convz, ub.gru.convr, ub.gru.convq, ub.motion_encoder.conv):
                conv.weight.mul_(3.0)
        elif regime == 'slope_gt1':
            cb.out_conv[2].weight.fill_(1.6)
    scale = (torch.rand(b, 1, 1, generator=g) * 3 + 0.5)
    y1 = (torch.randn(b, n, 128, generator=g) * scale + scale).to(dev)
    kfeat = torch.randn(b, n, 64, generator=g).to(dev)
    cflow = torch.randn(b, n, 64, generator=g).to(dev)
    flow = (0.3 * torch.randn(b, n, 3, generator=g)).to(dev)
    net = torch.tanh(torch.randn(b, n, 64, generator=g)).to(dev)
    inp = torch.relu(torch.randn(b, n, 64, generator=g)).to(dev)
    yd = y1.double().reshape(b, n, 8, 16)
    stats = torch.stack([yd.sum((1, 3)), (yd * yd).sum((1, 3))], -1).contiguous()   # [B,8,2]
    oc = cb.out_conv
    gn = dict(in_stats=stats, in_gamma=oc[1].weight.detach(), in_beta=oc[1].bias.detach(), in_count=float(n) * 16.0,
              in_act=2, in_slope=float(oc[2].weight.detach().reshape(-1)[0]))
    return y1, kfeat, cflow, flow, net, inp, gn


def unfused_chain(model, y1, kfeat, cflow, flow, net, inp, gn):
    from pvraft_b200 import ops
    me, ub = model.update_block.motion_encoder, model.update_block
    w_eff, b_eff = model.corr_block.corr_motion_weights(me)
    cc = ops.tc_linear([y1, kfeat], ops.tc_weights(w_eff), b_eff, out_act=ops.ACT_RELU, **gn)
    motion = ops.tc_linear([cc, cflow], ops.tc_weights(me.conv.weight), me.conv.bias.detach(), out_act=ops.ACT_RELU, tail=flow)
    net2 = ub.gru.forward_pm(net, inp, motion)
    sc = ub.flow_head.setconv
    p = ops.tc_linear([net2], ops.tc_weights(sc.fc1.weight, col0=0, cols=64))
    return net2, p


def fused_chain(model, y1, kfeat, cflow, flow, net, inp, gn):
    from pvraft_b200 import ops
    me, ub = model.update_block.motion_encoder, model.update_block
    gru, sc = ub.gru, ub.flow_head.setconv
    w_eff, b_eff = model.corr_block.corr_motion_weights(me)
    weights = (ops.tc_weights(w_eff), ops.tc_weights(me.conv.weight), ops.tc_weights((gru.convz.weight, gru.convr.weight)),
               ops.tc_weights(gru.convq.weight), ops.tc_weights(sc.fc1.weight, col0=0, cols=64))
    biases = (b_eff, me.conv.bias.detach(), gru.convz.bias.detach(), gru.convr.bias.detach(), gru.convq.bias.detach())
    return ops.update_chain(y1, gn, kfeat, cflow, flow, net, inp, weights, biases)


@pytest.mark.parametrize('shape', [(8, 8192), (5, 4096)], ids=['bench', 'multi_tile'])
@pytest.mark.parametrize('regime', ['random', 'trained', 'slope_gt1'])
def test_chain_kernel_bitwise(dev, shape, regime, monkeypatch):
    b, n = shape
    if shape == (5, 4096):   # more tiles than SMs: a CTA runs tiles of two samples
        assert b * n // 128 > torch.cuda.get_device_properties(dev).multi_processor_count
    model = make_model(dev, seed=3)
    y1, kfeat, cflow, flow, net, inp, gn = chain_inputs(model, b, n, dev, seed=11, regime=regime)
    want_net, want_p = unfused_chain(model, y1, kfeat, cflow, flow, net, inp, gn)
    empty_like = torch.empty_like
    monkeypatch.setattr(torch, 'empty_like', lambda t, *a, **k: empty_like(t, *a, **k).fill_(float('nan')))
    got_net, got_p = fused_chain(model, y1, kfeat, cflow, flow, net, inp, gn)
    monkeypatch.undo()
    torch.cuda.synchronize()
    assert torch.isfinite(want_net).all() and torch.isfinite(want_p).all()
    assert torch.equal(got_net, want_net)
    assert torch.equal(got_p, want_p)


@pytest.mark.parametrize('refine', [False, True], ids=['RSF', 'RSF_refine'])
@pytest.mark.parametrize('precision', ['fp32', 'bf16'])
def test_forward_fused_matches_unfused(dev, refine, precision, unfused):
    model = make_model(dev, refine=refine, seed=1)
    model.set_precision(precision)
    model.use_cuda_graph = False
    pc1, pc2 = clouds(2, 4096, 5, dev)
    with torch.no_grad():
        got = model([pc1, pc2], 4)
        with unfused:
            want = model([pc1, pc2], 4)
    got = got if isinstance(got, list) else [got]
    want = want if isinstance(want, list) else [want]
    assert len(got) == len(want)
    for a, b in zip(got, want):
        assert torch.equal(a, b)


def test_bench_shape_forward_and_launch_count(dev, unfused):
    from pvraft_b200 import ops
    model = make_model(dev, k=512, seed=2)
    model.use_cuda_graph = False
    pc1, pc2 = clouds(8, 8192, 7, dev)
    iters = 3
    with torch.no_grad():
        model([pc1, pc2], iters)                 # weight splits and derived constants
        l0 = ops.launch_count
        got = model([pc1, pc2], iters)
        fused = ops.launch_count - l0
        with unfused:
            model([pc1, pc2], iters)
            l0 = ops.launch_count
            want = model([pc1, pc2], iters)
            plain = ops.launch_count - l0
    assert plain - fused == 4 * iters
    for a, b in zip(got, want):
        assert torch.equal(a, b)


def test_graph_replay_matches_eager_deterministic(dev):
    model = make_model(dev, seed=4)
    pc1, pc2 = clouds(2, 2048, 9, dev)
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        with torch.no_grad():
            model.use_cuda_graph = False
            eager = model([pc1, pc2], 3)
            model.use_cuda_graph = True
            replay = model([pc1, pc2], 3)
            replay2 = model([pc1, pc2], 3)
    finally:
        torch.use_deterministic_algorithms(old)
    for a, b, c in zip(eager, replay, replay2):
        assert torch.equal(a, b) and torch.equal(a, c)
