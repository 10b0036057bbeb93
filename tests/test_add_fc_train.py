"""TrainStep (legacy executor) with stacked shared layers (add_fc 2 and 3).

CPU: the extra layers' slots sit in the late part of the flat bucket; phased mode, class weights and the DANN schedule
are refused.  GPU: one step against the fp64 oracle with dropout off and on (the per-layer masks rebuilt from the
counter RNG), eager == graph and reruns bit for bit, the device sampler == load(), three SGD and Adam steps against the
stock autograd loop on VideoModel, resume from state_dict(), MCD at mu 0 and 0.7 with the meters.
"""
import copy

import pytest
import torch

from oracle import add_fc_oracle as afo
from oracle import ta3n_oracle as orc
from tests.golden_util import assert_close

gpu = pytest.mark.gpu
BETA = (0.75, 0.6, 0.5)
GRAD_TOL = {"fp32": 4e-4, "tf32x3": 1e-3}
NOISE_SCALE = {"fp32": 1.0, "tf32x3": 8.0}


def _model(add_fc, T=5, C=7, fc_dim=256, drop=0.0, attn_frame="none", ens="none", device="cpu", seed=3):
    from ta3n_b200.models import VideoModel
    torch.manual_seed(seed)
    m = VideoModel(C, "video", "trn-m", "RGB", train_segments=T, val_segments=T, add_fc=add_fc, fc_dim=fc_dim,
                   dropout_i=drop, dropout_v=drop, partial_bn=False, use_attn_frame=attn_frame, ens_DA=ens,
                   verbose=False)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for k, v in sorted(m.named_parameters()):
            if k.endswith("weight"):
                v.add_(0.02 * torch.randn(v.shape, generator=g))
    return m.to(device).train()


# ---- CPU -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("add_fc", [1, 2, 3])
@pytest.mark.parametrize("ens", ["none", "MCD"])
def test_bucket_layout_puts_the_stacked_layers_late(add_fc, ens):
    from ta3n_b200.train import _N_LATE, bucket_layout, stack_slots, step_parameters
    m = _model(add_fc, ens=ens)
    params = step_parameters(m)
    stack = stack_slots(m)
    assert len(stack) == 2 * (add_fc - 1)
    assert [params[i] for i in stack] == m.path_parameters()[len(m.path_parameters()) - len(stack):]
    order, offs, total, early = bucket_layout(params, stack)
    assert sorted(order) == list(range(len(params)))
    late = order[len(order) - _N_LATE - len(stack):]
    if add_fc == 1:
        assert late == list(range(_N_LATE)) and order == bucket_layout(params)[0]
    else:
        # completion order: frame disc, shared_3, shared_2, shared_1
        layers = [stack[i:i + 2] for i in range(0, len(stack), 2)]
        assert late == [2, 3, 4, 5] + [i for pair in reversed(layers) for i in pair] + [0, 1]
    assert all(offs[i] >= early for i in late) and all(offs[i] < early for i in order[:len(order) - len(late)])


def test_train_step_refusals_with_stacked_layers():
    from ta3n_b200.train import TrainStep
    m = _model(2)
    with pytest.raises(NotImplementedError, match="legacy"):
        TrainStep(m, 4, 4, BETA, mode="phased")
    with pytest.raises(NotImplementedError, match="add_fc"):
        TrainStep(m, 4, 4, BETA, class_weight=torch.ones(7))
    with pytest.raises(NotImplementedError, match="add_fc"):
        TrainStep(m, 4, 4, (0.75, -1.0, 0.5))
    with pytest.raises(NotImplementedError, match="add_fc"):
        TrainStep(m, 4, 4, BETA, domain_weight=(1.0, 2.0))


# ---- GPU -----------------------------------------------------------------------------------------------------------
def _inputs(bs, bt, T, seed=9):
    g = torch.Generator().manual_seed(seed)
    xs = torch.randn(bs, T, orc.FEATURE_DIM, generator=g)
    xt = torch.randn(bt, T, orc.FEATURE_DIM, generator=g) - 0.2
    return xs, xt, torch.arange(bs) % 7


def _engine(name):
    import ta3n_b200
    ta3n_b200.set_gemm_engine(name)


@pytest.fixture(params=["fp32", "tf32x3"])
def engine(request):
    _engine(request.param)
    yield request.param
    _engine("tf32x3")


@gpu
@pytest.mark.parametrize("add_fc,attn_frame,drop", [(2, "none", 0.0), (3, "none", 0.0), (2, "TransAttn", 0.5),
                                                    (3, "none", 0.5)])
def test_train_step_matches_fp64_oracle(add_fc, attn_frame, drop, engine):
    """One TrainStep against the fp64 oracle: loss and every gradient; with dropout on, the oracle takes the masks
    of every shared layer and of dropout_v rebuilt from the counter RNG with the step's per-layer seeds (the fp64
    ReLU pattern; these engines are fp32 grade in the forward)."""
    from ta3n_b200.train import TrainStep
    T, bs, bt = 5, 10, 7
    m = _model(add_fc, T=T, drop=drop, attn_frame=attn_frame, device="cuda")
    cfg = orc.PathConfig(num_class=7, num_segments=T, fc_dim=256, dropout_i=drop, dropout_v=drop,
                         use_attn_frame=attn_frame)
    params = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    xs, xt, labels = _inputs(bs, bt, T)
    step = TrainStep(m, bs, bt, BETA, use_graph=False)
    loss = step(xs.pin_memory(), xt.pin_memory(), labels)
    torch.cuda.synchronize()
    masks = None
    if drop > 0:
        masks = afo.train_step_masks(int(step.step_counter.item()), bs, bt, T, cfg.shared_dim, cfg.video_dim, drop,
                                     drop, add_fc)
    p64 = {k: v.double() if v.dtype.is_floating_point else v for k, v in params.items()}
    gates = afo.activation_pattern(p64, xs.double(), xt.double(), BETA, cfg, add_fc, masks)
    l64, _, g64 = afo.train_step(p64, xs.double(), xt.double(), labels, BETA, cfg, add_fc, train=drop > 0,
                                 masks=masks, gates=gates)
    _, _, g32 = afo.train_step(params, xs, xt, labels, BETA, cfg, add_fc, train=drop > 0, masks=masks, gates=gates)
    assert_close(loss.cpu()[0], l64, 2e-4, "loss")
    named = dict(m.named_parameters())
    for name, g in g64.items():
        if g is None:
            continue
        noise = (g32[name].double() - g).norm().item() * NOISE_SCALE[engine]
        assert_close(named[name].grad, g, GRAD_TOL[engine], f"grad {name}", noise=noise)


@gpu
@pytest.mark.parametrize("add_fc", [2, 3])
def test_eager_and_graph_are_bit_identical(add_fc):
    """The same three SGD steps eagerly and through the captured graph (dropout off: the capture's warm-up advances
    the dropout counter), then the graph again with dropout on, twice: bit for bit."""
    from ta3n_b200.train import SGDNesterov, TrainStep
    xs, xt, labels = _inputs(6, 5, 5)
    runs = []
    for use_graph, drop in ((False, 0.0), (True, 0.0), (True, 0.5), (True, 0.5)):
        m = _model(add_fc, drop=drop, device="cuda")
        step = TrainStep(m, 6, 5, BETA, use_graph=use_graph, optimizer=SGDNesterov(lr=0.01), seed=11)
        losses = [step(xs, xt, labels).clone() for _ in range(3)]
        torch.cuda.synchronize()
        runs.append((torch.cat(losses), step.flat_param.clone(), step.flat_grad.clone()))
    assert all(torch.equal(a, b) for a, b in zip(runs[0], runs[1]))
    assert all(torch.equal(a, b) for a, b in zip(runs[2], runs[3]))
    assert not torch.equal(runs[1][0], runs[2][0])


def _stock_loop(m, xs, xt, labels, opt_name, n):
    """main.py's iteration on VideoModel through autograd: loss, backward, clip_grad_norm_, torch.optim."""
    from ta3n_b200.loss import ta3n_loss
    params = [p for p in m.parameters()]
    opt = torch.optim.SGD(params, 0.01, momentum=0.9, weight_decay=1e-4, nesterov=True) if opt_name == "sgd" else \
        torch.optim.Adam(params, 1e-3, weight_decay=1e-4)
    d = torch.device("cuda")
    for _ in range(n):
        opt.zero_grad(set_to_none=True)
        outs = m(xs.to(d), xt.to(d), list(BETA), 0, is_train=True, reverse=False)
        loss = ta3n_loss(outs, labels.to(d), 0.003)
        loss.backward()
        torch.nn.utils.clip_grad_norm_([p for p in params if p.grad is not None], 20.0)
        opt.step()


@gpu
@pytest.mark.parametrize("opt_name", ["sgd", "adam"])
def test_three_steps_match_the_stock_autograd_loop(opt_name):
    """Three SGD-Nesterov / Adam steps of TrainStep (add_fc=3, dropout off) against VideoModel + autograd +
    torch.optim: every parameter within 1e-4 (relative, normwise)."""
    from ta3n_b200.train import Adam, SGDNesterov, TrainStep
    xs, xt, labels = _inputs(8, 6, 5)
    m_a = _model(3, device="cuda")
    m_b = copy.deepcopy(m_a)
    opt = SGDNesterov(lr=0.01) if opt_name == "sgd" else Adam(lr=1e-3)
    step = TrainStep(m_a, 8, 6, BETA, optimizer=opt)
    for _ in range(3):
        step(xs, xt, labels)
    torch.cuda.synchronize()
    _stock_loop(m_b, xs, xt, labels, opt_name, 3)
    pb = dict(m_b.named_parameters())
    for name, p in m_a.named_parameters():
        assert_close(p.detach(), pb[name].detach(), 1e-4, name)


@gpu
def test_resume_from_state_dict_is_bit_identical():
    from ta3n_b200.train import Adam, TrainStep
    xs, xt, labels = _inputs(6, 5, 5)
    m_a = _model(2, drop=0.5, device="cuda")
    m_b = copy.deepcopy(m_a)
    a = TrainStep(m_a, 6, 5, BETA, optimizer=Adam(lr=1e-3), seed=5)
    for _ in range(4):
        a(xs, xt, labels)
    b0 = TrainStep(m_b, 6, 5, BETA, optimizer=Adam(lr=1e-3), seed=5)
    for _ in range(2):
        b0(xs, xt, labels)
    sd = copy.deepcopy(b0.state_dict())
    params = copy.deepcopy(m_b.state_dict())
    m_c = _model(2, drop=0.5, device="cuda", seed=99)
    m_c.load_state_dict(params)
    c = TrainStep(m_c, 6, 5, BETA, optimizer=Adam(lr=1e-3), seed=5)
    c.load_state_dict(sd)
    for _ in range(2):
        c(xs, xt, labels)
    torch.cuda.synchronize()
    assert torch.equal(a.flat_param, c.flat_param)


@gpu
def test_device_sampler_equals_load(tmp_path):
    """The device sampler's gather and the host load() give the same steps bit for bit, the last batch short."""
    from ta3n_b200 import dataset as D
    from ta3n_b200.train import SGDNesterov, TrainStep
    from tests.test_device_sampler import _banks
    batch = (4, 4)
    sets, banks = _banks(tmp_path, 5, 2048, (10, None), (9, None), batch)
    m_a = _model(3, drop=0.5, device="cuda")
    m_b = copy.deepcopy(m_a)
    sampler = D.DevicePairedSampler(banks[0], banks[1], batch, seed=4)
    step_a = TrainStep(m_a, *batch, BETA, sampler=sampler, optimizer=SGDNesterov(lr=0.01), seed=7)
    step_b = TrainStep(m_b, *batch, BETA, optimizer=SGDNesterov(lr=0.01), seed=7)
    loader = D.PairedFeatureLoader(sets[0], sets[1], batch, seed=4)
    assert sampler.start_epoch() == len(loader)
    for (xs, ys), (xt, _) in loader:
        if xs.shape[0] < batch[0] or xt.shape[0] < batch[1]:
            step_b.xs.zero_(), step_b.xt.zero_(), step_b.labels.zero_()
        step_b.load(xs, xt, ys)
        lb = step_b.run().clone()
        la = step_a.run().clone()
        torch.cuda.synchronize()
        assert torch.equal(la, lb) and torch.isfinite(la).all()
        assert torch.equal(step_a.flat_param, step_b.flat_param)


@gpu
@pytest.mark.parametrize("mu", [0.0, 0.7])
def test_mcd_with_stacked_layers(mu):
    """ens_DA='MCD' at add_fc=2: the two passes in one graph equal the eager sequence bit for bit (dropout off), a
    graph with dropout on reruns bit for bit with pass 2 on its own per-layer seeds, and the meters (stats=True) hold
    the loss the step reports."""
    from ta3n_b200.train import SGDNesterov, TrainStep
    xs, xt, labels = _inputs(6, 5, 5)
    res = []
    for use_graph, drop in ((False, 0.0), (True, 0.0), (True, 0.5), (True, 0.5)):
        m = _model(2, drop=drop, ens="MCD", device="cuda")
        step = TrainStep(m, 6, 5, BETA, mu=mu, use_graph=use_graph, optimizer=SGDNesterov(lr=0.01), stats=True,
                         seed=13)
        losses = torch.cat([step(xs, xt, labels).clone() for _ in range(2)])
        st = step.stats()
        res.append((losses, step.flat_param.clone(), st.loss.sum))
        assert torch.isfinite(losses).all()
        assert st.steps == 2 and st.loss.val == pytest.approx(float(losses[-1]), rel=1e-6)
        if drop > 0:
            assert step.spec2.drop_stack[0].seed != step.spec.drop_stack[0].seed
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
    assert torch.equal(res[2][0], res[3][0]) and torch.equal(res[2][1], res[3][1])


FULL = {"cfg2_fc2": (256, 256, 5, 12, "none", 2), "cfg2_fc3": (256, 256, 5, 12, "none", 3),
        "cfg3_fc2": (128, 128, 9, 12, "TransAttn", 2), "small_fc3": (24, 20, 5, 12, "none", 3)}


@gpu
@pytest.mark.parametrize("eng", ["fp32", "tf32x3", "tf32"])
@pytest.mark.parametrize("name", list(FULL))
def test_step_on_realised_pattern(name, eng):
    """TrainStep (dropout off, fc_dim 512) against the fp64 oracle -- run on the GPU -- evaluated on the ReLU pattern
    the step realised in every layer (every shared layer, frame discriminator, TRN, relation and video
    discriminators).  Units whose state differs from the fp64 pattern, counted over every shared layer: at most 5e-6
    of them on the fp32-grade engines, 2e-3 under plain tf32.  Every gradient within 1e-3 (3e-3 under plain tf32)
    plus the rounding-noise allowance."""
    from ta3n_b200.train import TrainStep
    bs, bt, T, C, attn_frame, L = FULL[name]
    if name.startswith("cfg") and eng == "tf32":
        pytest.skip("plain tf32 is held to the pinned pattern on the small case")
    _engine(eng)
    try:
        torch.manual_seed(1)
        m = _model(L, T=T, C=C, fc_dim=512, attn_frame=attn_frame, device="cuda", seed=21)
        cfg = orc.PathConfig(num_class=C, num_segments=T, fc_dim=512, dropout_i=0.0, dropout_v=0.0,
                             use_attn_frame=attn_frame)
        params = {k: v.detach().clone() for k, v in m.state_dict().items()}
        g = torch.Generator().manual_seed(2)
        xs = torch.randn(bs, T, orc.FEATURE_DIM, generator=g)
        xt = torch.randn(bt, T, orc.FEATURE_DIM, generator=g) + 0.1
        labels = torch.arange(bs) % C
        step = TrainStep(m, bs, bt, BETA, use_graph=False)
        loss = step(xs, xt, labels)
        torch.cuda.synchronize()
        pool = step.bufs.pool
        shared_keys = ["shared"] + [f"shared{layer}" for layer in range(2, L + 1)]
        feats = [pool[f"feat_{layer}"] for layer in range(1, L)] + [pool["feat"]]
        gates = {k: (f > 0).cpu() for k, f in zip(shared_keys, feats)}
        gates.update({"frame_disc": (pool["hid_f"] > 0).cpu(), "trn": [(a > 0).cpu() for a in pool["act"]],
                      "rel_disc": [(h > 0).cpu() for h in pool["hid_r"]], "video_disc": (pool["hid_v"] > 0).cpu()})
        params = {k: v.cpu() for k, v in params.items()}
        p64 = {k: v.double() if v.dtype.is_floating_point else v for k, v in params.items()}
        x64s, x64t = xs.double(), xt.double()
        plain = afo.activation_pattern(p64, x64s, x64t, BETA, cfg, L)
        flips = sum(int((gates[k] != plain[k]).sum()) for k in shared_keys)
        total = sum(gates[k].numel() for k in shared_keys)
        bound = 2e-3 if eng == "tf32" else 5e-6
        assert flips <= bound * total, f"{flips} of {total} shared units changed state"
        l64, _, g64 = afo.train_step(p64, x64s, x64t, labels, BETA, cfg, L, gates=gates)
        _, _, g32 = afo.train_step(params, xs, xt, labels, BETA, cfg, L, gates=gates)
        tol = 3e-3 if eng == "tf32" else 1e-3
        assert_close(loss.cpu()[0], l64, tol, "loss")
        named = dict(m.named_parameters())
        scale = {"fp32": 1.0, "tf32x3": 8.0, "tf32": 2.0 ** 13}[eng]
        for k, go in g64.items():
            if go is None:
                continue
            assert_close(named[k].grad, go, tol, f"grad {k}", noise=(g32[k].double() - go).norm().item() * scale)
    finally:
        _engine("tf32x3")
