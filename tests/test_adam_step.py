"""TrainStep(optimizer=Adam(...)) and optimizer checkpoints on the GPU.

Adam turns gradient rounding noise into full-size updates (its first step moves every element by about lr whatever
the size of its gradient), so a step is checked in two halves rather than end to end against the fp64 oracle:
  (a) the gradient the step wrote (flat_grad, which the update leaves unchanged) against the oracle's gradient at the
      pre-step parameters, with the tolerances of tests/test_gpu_parity.py;
  (b) the parameter and moment update against fp64 clip + Adam applied to that same GPU gradient, from the pre-step
      parameters and state, at a tight tolerance.
Also: the kernel against torch.optim.Adam in fp64, graph replays against eager calls, hand-over of the state to and from
stock torch.optim optimizers, and a resumed run against an uninterrupted one, bit for bit.
"""
import io

import pytest
import torch

from oracle import ta3n_oracle as orc
from tests import optim_oracle as oo
from tests.golden_util import assert_close

pytestmark = pytest.mark.gpu
BETA = (0.75, 0.75, 0.5)


def _dev():
    return torch.device("cuda:0")


@pytest.fixture(params=["fp32", "tf32x3", "tf32"])
def engine(request):
    import ta3n_b200
    ta3n_b200.set_gemm_engine(request.param)
    yield request.param
    ta3n_b200.set_gemm_engine("tf32x3")


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------
# the kernel
# ------------------------------------------------------------------------------------------------
class _Flat:
    """Flat device buffers for ta3n_adam_step_masked."""

    def __init__(self, p, active=None):
        from ta3n_b200 import _lib
        self.lib = _lib.load()
        n = p.numel()
        self.n = n
        self.p = p.to(_dev()).contiguous()
        self.m = torch.zeros(n, device=_dev())
        self.v = torch.zeros(n, device=_dev())
        self.lr = torch.zeros(1, device=_dev())
        self.t = torch.zeros(1, device=_dev(), dtype=torch.int64)
        self.stats = torch.zeros(2, device=_dev())
        self.ws = torch.zeros(self.lib.ta3n_adam_workspace_bytes() // 4 + 1, device=_dev())
        self.active = None if active is None else active.to(_dev()).contiguous()

    def step(self, g, max_norm, betas=(0.9, 0.999), eps=1e-8, wd=1e-3):
        from ta3n_b200 import _lib
        _lib.check(self.lib.ta3n_adam_step_masked(
            self.p.data_ptr(), g.data_ptr(), self.m.data_ptr(), self.v.data_ptr(), self.n, self.lr.data_ptr(),
            self.t.data_ptr(), betas[0], betas[1], eps, wd, max_norm, self.ws.data_ptr(), self.ws.numel() * 4,
            self.stats.data_ptr(), None if self.active is None else self.active.data_ptr(), _stream()))


def _mask(n, seed):
    """A per-element mask, constant over aligned groups of four (the entry's contract), about a third masked."""
    g = torch.Generator().manual_seed(seed)
    groups = (torch.rand(-(-n // 4), generator=g) > 0.33).float()
    groups[0] = 1.0
    return groups.repeat_interleave(4)[:n]


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("clip", ["active", "inactive", "off"])
@pytest.mark.parametrize("n", [1000003, 4096, 7])
def test_adam_kernel_matches_torch_optim(n, clip, masked):
    """Five steps with a changing lr against clip_grad_norm_ + torch.optim.Adam in fp64 on the same buffers.  The
    masked elements play parameters whose .grad is None: torch leaves them alone, and so must the kernel.  The norm and
    coefficient the kernel reports are checked as for SGD; the fp64 update then uses the kernel's coefficient, so that
    the comparison of the update measures the update alone.  Gradients are O(1), so their squares are normal fp32."""
    g = torch.Generator().manual_seed(n + 7)
    p0 = torch.randn(n, generator=g)
    active = _mask(n, n) if masked else None
    on = torch.ones(n, dtype=torch.bool) if active is None else active.bool()
    ref = torch.nn.Parameter(p0[on].double())
    opt = torch.optim.Adam([ref], 0.01, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-3, foreach=False)
    buf = _Flat(p0, active)
    max_norm = {"active": 0.5, "inactive": 1e9, "off": 0.0}[clip]
    for it in range(5):
        grad = torch.randn(n, generator=g) * (1.0 + it)
        lr_it = 0.01 / (1 + it)
        opt.param_groups[0]["lr"] = lr_it
        buf.lr.fill_(lr_it)
        buf.step(grad.to(_dev()), max_norm)
        torch.cuda.synchronize()
        coef = 1.0
        if max_norm > 0:
            norm_ref = grad.double().norm()            # clip_grad_norm_ runs over every gradient, masked ones too
            assert_close(buf.stats[0].cpu(), norm_ref, 2e-6, "total norm")
            want = min(1.0, max_norm / (float(norm_ref) + 1e-6))
            assert abs(float(buf.stats[1]) - want) < 1e-6 * max(1.0, want)
            coef = float(buf.stats[1])
            assert (coef < 1.0) == (clip == "active")
        ref.grad = grad[on].double() * coef
        opt.step()
        assert int(buf.t.item()) == it + 1
    st = opt.state[ref]
    assert_close(buf.p.cpu()[on], ref.detach(), 1e-6, "parameters")
    assert_close(buf.p.cpu()[on].double() - p0[on].double(), ref.detach() - p0[on].double(), 1e-5, "update")
    assert_close(buf.m.cpu()[on], st["exp_avg"], 1e-6, "exp_avg")
    assert_close(buf.v.cpu()[on], st["exp_avg_sq"], 1e-6, "exp_avg_sq")
    if masked:
        assert torch.equal(buf.p.cpu()[~on], p0[~on])
        assert not buf.m.cpu()[~on].any() and not buf.v.cpu()[~on].any()


def test_adam_kernel_keeps_zero_gradients_and_parameters_at_zero():
    """The padding between slots of the flat buffers: p = g = m = v = 0 must stay exactly 0 (0 / eps = 0)."""
    buf = _Flat(torch.zeros(4096))
    buf.lr.fill_(0.1)
    zeros = torch.zeros(4096, device=_dev())
    for _ in range(3):
        buf.step(zeros, 0.5)
    torch.cuda.synchronize()
    assert not buf.p.any() and not buf.m.any() and not buf.v.any()
    assert int(buf.t.item()) == 3 and float(buf.stats[0]) == 0.0 and float(buf.stats[1]) == 1.0


@pytest.mark.parametrize("masked", [False, True])
def test_adam_graph_replays_equal_eager_calls(masked):
    """N replays of one captured graph (lr changed between replays, outside the graph) equal N eager calls bit for
    bit, step count included: the count advances inside the kernel."""
    n = 100003
    g = torch.Generator().manual_seed(5)
    p0 = torch.randn(n, generator=g)
    grads = [torch.randn(n, generator=g).to(_dev()) * (1 + k) for k in range(5)]
    active = _mask(n, 3) if masked else None
    eager, graphed = _Flat(p0, active), _Flat(p0, active)
    gin = torch.zeros(n, device=_dev())
    _Flat(torch.zeros(8)).step(torch.zeros(8, device=_dev()), 1.0)      # the kernels are loaded before the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        graphed.step(gin, 2.0)
    torch.cuda.synchronize()
    assert int(graphed.t.item()) == 0            # capturing runs nothing
    for k, gr in enumerate(grads):
        lr = 0.01 / (1 + k)
        eager.lr.fill_(lr)
        eager.step(gr, 2.0)
        graphed.lr.fill_(lr)
        gin.copy_(gr)
        graph.replay()
    torch.cuda.synchronize()
    for a, b in ((eager.p, graphed.p), (eager.m, graphed.m), (eager.v, graphed.v), (eager.t, graphed.t),
                 (eager.stats, graphed.stats)):
        assert torch.equal(a, b)
    assert int(graphed.t.item()) == 5


# ------------------------------------------------------------------------------------------------
# TrainStep(optimizer=Adam)
# ------------------------------------------------------------------------------------------------
def _flat_snapshot(step):
    out = {"p": step.flat_param.detach().double().cpu(), "g": step.flat_grad.detach().double().cpu()}
    if hasattr(step, "exp_avg"):
        out.update(m=step.exp_avg.double().cpu(), v=step.exp_avg_sq.double().cpu(), t=int(step.adam_step.item()))
    else:
        out.update(m=step.momentum_buf.double().cpu())
    return out


def _reference_update(step, pre, g, lr):
    """fp64 clip_grad_norm_ + the configured update, as the oracle states them (``oracle.ta3n_oracle.clip_grad_norm`` /
    ``sgd_nesterov_step``, ``tests.optim_oracle.adam_step``), applied to the GPU's gradient `g` from the pre-step state.
    Masked elements are parameters without a gradient, which torch leaves alone."""
    from ta3n_b200.train import Adam
    o = step.opt
    keep = torch.zeros_like(g, dtype=torch.bool) if step.active_mask is None else (step.active_mask.cpu() == 0)
    on = ~keep
    grads = {"flat": g.clone()}
    if o.clip_gradient is not None:
        orc.clip_grad_norm(grads, o.clip_gradient)        # over every element, as clip_grad_norm_(model.parameters())
    params, grads = {"flat": pre["p"][on].clone()}, {"flat": grads["flat"][on]}
    if isinstance(o, Adam):
        state = {"flat": {"step": pre["t"], "exp_avg": pre["m"][on].clone(), "exp_avg_sq": pre["v"][on].clone()}}
        oo.adam_step(params, grads, state, lr, tuple(o.betas), o.eps, o.weight_decay)
        upd = {"p": params["flat"], "m": state["flat"]["exp_avg"], "v": state["flat"]["exp_avg_sq"]}
    else:
        bufs = {"flat": pre["m"][on].clone()}
        orc.sgd_nesterov_step(params, grads, bufs, lr, o.momentum, o.weight_decay)
        upd = {"p": params["flat"], "m": bufs["flat"]}
    new = {}
    for k, x in upd.items():
        new[k] = pre[k].clone()
        new[k][on] = x
    return new, keep


def _check_update(step, pre, lr, what):
    """Half (b): the update the step applied against fp64 clip + update on the GPU's own gradient."""
    post = _flat_snapshot(step)
    want, keep = _reference_update(step, pre, post["g"], lr)
    noise = 3 * 6e-8 * pre["p"].norm().item()           # fp32 storage of the parameters
    assert_close(post["p"] - pre["p"], want["p"] - pre["p"], 1e-5, f"{what}: update", noise=noise)
    for k in want:
        if k != "p":
            assert_close(post[k], want[k], 1e-5, f"{what}: {k}")
        assert torch.equal(post[k][keep], pre[k][keep]), f"{what}: masked {k} moved"
    if "t" in pre:
        assert post["t"] == pre["t"] + 1


def _state_cpu(model):
    return {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}


def _plain_case(seed=33, C=5, bs=12, bt=7, dropout=0.0):
    cfg = orc.PathConfig(num_class=C, num_segments=5, fc_dim=512, dropout_i=dropout, dropout_v=dropout)
    params = orc.init_params(cfg, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    for k in params:
        if params[k].dtype.is_floating_point and k.startswith(orc.USED_PARAM_PREFIXES) and "weight" in k:
            params[k] = params[k] + 0.02 * torch.randn(params[k].shape, generator=g)
    xs = torch.randn(bs, 5, orc.FEATURE_DIM, generator=g)
    xt = torch.randn(bt, 5, orc.FEATURE_DIM, generator=g) - 0.2
    labels = torch.arange(bs) % C
    return cfg, params, xs, xt, labels


def _check_plain_gradients(step, params_pre, cfg, xs, xt, labels, engine, what):
    """Half (a) for the plain step: p.grad against the fp64 oracle at the pre-step parameters."""
    from tests.test_gpu_parity import GRAD_TOL, NOISE_SCALE, oracle_truth
    _, _, g64, _, _, n_grad = oracle_truth(params_pre, xs, xt, labels, BETA, cfg, 0.003, True, None)
    named = dict(step.model.named_parameters())
    for name, go in g64.items():
        assert_close(named[name].grad, go, GRAD_TOL[engine], f"{what}: grad {name}",
                     noise=n_grad[name] * NOISE_SCALE[engine])


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("mode", ["legacy", "phased"])
def test_train_step_adam_iterations(mode, use_graph, engine):
    """Three iterations with a DANN learning rate: gradients against the oracle, updates against fp64 Adam."""
    from ta3n_b200.train import Adam, TrainStep, lr_dann
    from tests.test_gpu_parity import build_model
    cfg, params, xs, xt, labels = _plain_case()
    model = build_model(cfg, params, train=True)
    lr0 = 0.002
    step = TrainStep(model, xs.shape[0], xt.shape[0], BETA, gamma=0.003, use_graph=use_graph, mode=mode,
                     optimizer=Adam(lr=lr0, weight_decay=1e-4, clip_gradient=10.0))
    for it in range(3):
        lr = lr_dann(lr0, it / 3.0)
        step.set_lr(lr)
        params_pre = _state_cpu(model)
        pre = _flat_snapshot(step)
        step(xs.pin_memory(), xt.pin_memory(), labels)
        torch.cuda.synchronize()
        what = f"{mode} graph={use_graph} iteration {it}"
        _check_plain_gradients(step, params_pre, cfg, xs, xt, labels, engine, what)
        _check_update(step, pre, lr, what)
    assert torch.equal(model.fc_feature_source.weight.detach().cpu(), params["fc_feature_source.weight"])


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("mu", [0.0, 0.7])
def test_mcd_train_step_adam_iterations(mu, use_graph, engine):
    from ta3n_b200.train import Adam, TrainStep, lr_dann
    from tests.test_gpu_parity import build_model
    from tests.test_mcd_train_step import BETA as MBETA, _check_mcd_step, _gpu_case
    cfg, params, xs, xt, labels, _ = _gpu_case("attn_t5_mu0")
    model = build_model(cfg, params, train=True)
    lr0 = 0.002
    step = TrainStep(model, xs.shape[0], xt.shape[0], MBETA, gamma=0.003, use_graph=use_graph, mu=mu,
                     optimizer=Adam(lr=lr0, clip_gradient=5.0))
    for it in range(3):
        lr = lr_dann(lr0, it / 3.0)
        step.set_lr(lr)
        params_pre = _state_cpu(model)
        pre = _flat_snapshot(step)
        loss = step(xs.to(_dev()), xt.to(_dev()), labels.to(_dev()))
        torch.cuda.synchronize()
        what = f"MCD mu={mu} graph={use_graph} iteration {it}"
        _check_mcd_step(step, None, loss.cpu()[0], cfg, params_pre, xs, xt, labels, mu, engine, what)
        _check_update(step, pre, lr, what)
    assert not torch.equal(model.fc_classifier_video_source_2.weight.detach().cpu(),
                           params["fc_classifier_video_source_2.weight"])


def test_adam_leaves_parameters_without_gradient_alone():
    """place_adv[2] = 'N': the frame discriminator gets no gradient, so torch.optim.Adam never touches it (no decay,
    no state); the fused update must not either, and the exported state has no entry for it."""
    from ta3n_b200.train import Adam, TrainStep
    from tests.test_gpu_parity import build_model
    cfg, params, xs, xt, labels = _plain_case(seed=3)
    model = build_model(cfg, params, train=True)
    eager = TrainStep(build_model(cfg, params, train=True), 12, 7, BETA, use_graph=False, place_adv=("Y", "Y", "N"),
                      optimizer=Adam(lr=0.01, weight_decay=0.1))
    step = TrainStep(model, 12, 7, BETA, use_graph=True, place_adv=("Y", "Y", "N"),
                     optimizer=Adam(lr=0.01, weight_decay=0.1))
    before = {k: p.detach().clone() for k, p in model.named_parameters()}
    for _ in range(3):
        step(xs, xt, labels)
        eager(xs, xt, labels)
    torch.cuda.synchronize()
    assert eager.launches_per_step == step.launches_per_step      # the graph's count includes the optimizer's
    after = dict(model.named_parameters())
    frame = ("fc_feature_domain.weight", "fc_feature_domain.bias", "fc_classifier_domain.weight",
             "fc_classifier_domain.bias")
    for name in frame:
        assert torch.equal(after[name].detach(), before[name]), name
    assert not torch.equal(after["fc_feature_shared_source.weight"].detach(), before["fc_feature_shared_source.weight"])
    sd = step.optimizer_state_dict()
    index = {n: i for i, (n, _) in enumerate(model.named_parameters())}
    assert not any(index[n] in sd["state"] for n in frame)
    assert all(float(e["step"]) == 3.0 for e in sd["state"].values())


# ------------------------------------------------------------------------------------------------
# hand-over to and from stock torch.optim
# ------------------------------------------------------------------------------------------------
def _stock_optimizer(model, kind, lr):
    if kind == "adam":
        return torch.optim.Adam(model.parameters(), lr, weight_decay=1e-4)
    return torch.optim.SGD(model.parameters(), lr, momentum=0.9, weight_decay=1e-4, nesterov=True)


def _stock_iterations(model, opt, xs, xt, labels, k):
    """main.py:418-583 as the reference runs it: autograd forward and backward, clip_grad_norm_, optimizer.step()."""
    from ta3n_b200.loss import ta3n_loss
    for _ in range(k):
        outs = model(xs, xt, list(BETA), 0, is_train=True, reverse=False)
        loss = ta3n_loss(outs, labels, 0.003)
        opt.zero_grad()
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), 20.0)
        opt.step()


def _assert_state_equals_flat(step, opt, what):
    """Every stock state tensor equals its slot of the flat buffers bit for bit; no other slot holds state."""
    from ta3n_b200.train import bucket_layout
    names = {"exp_avg": "exp_avg", "exp_avg_sq": "exp_avg_sq", "momentum_buffer": "momentum_buf"}
    _, offs, _, _ = bucket_layout(step.params)
    held = 0
    for j, p in enumerate(step.params):
        st = opt.state.get(p)
        if not st:
            continue
        held += 1
        for k, attr in names.items():
            if k in st:
                flat = getattr(step, attr)[offs[j]:offs[j] + p.numel()].view_as(p)
                assert torch.equal(st[k].to(flat.device), flat), f"{what}: {k} of parameter {j}"
        if "step" in st:
            assert int(float(st["step"])) == int(step.adam_step.item()), what
    assert held == len(opt.state), f"{what}: state for parameters outside the flat buffers"


@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_state_hands_over_between_stock_torch_and_train_step(kind):
    from ta3n_b200.train import Adam, SGDNesterov, TrainStep
    from tests.test_gpu_parity import build_model
    cfg, params, xs, xt, labels = _plain_case(seed=11)
    dev = _dev()
    xs, xt, labels = xs.to(dev), xt.to(dev), labels.to(dev)
    lr = 0.001
    # stock loop for k = 2 steps, then TrainStep continues it
    model = build_model(cfg, params, train=True)
    stock = _stock_optimizer(model, kind, lr)
    _stock_iterations(model, stock, xs, xt, labels, 2)
    stock_keys = stock.state_dict()
    opt_cfg = Adam(lr=0.5) if kind == "adam" else SGDNesterov(lr=0.5)      # lr comes from the loaded dict
    step = TrainStep(model, xs.shape[0], xt.shape[0], BETA, gamma=0.003, optimizer=opt_cfg)
    step.load_optimizer_state_dict(stock.state_dict())
    assert step.opt.lr == lr and float(step.lr_dev) == torch.tensor(lr, dtype=torch.float32).item()
    torch.cuda.synchronize()
    _assert_state_equals_flat(step, stock, "stock -> TrainStep")
    pre = _flat_snapshot(step)
    step(xs, xt, labels)
    torch.cuda.synchronize()
    _check_update(step, pre, lr, "first fused update after the hand-over")
    # and back: TrainStep's state into a stock optimizer
    step(xs, xt, labels)
    sd = step.optimizer_state_dict()
    fresh = _stock_optimizer(model, kind, 0.5)
    fresh.load_state_dict(sd)
    _assert_state_equals_flat(step, fresh, "TrainStep -> stock")
    assert fresh.param_groups[0]["lr"] == lr
    # the same keys as the stock loop's
    assert sd.keys() == stock_keys.keys() and sd["state"].keys() == stock_keys["state"].keys()
    assert sd["param_groups"][0].keys() == stock_keys["param_groups"][0].keys()
    for i, e in stock_keys["state"].items():
        assert list(sd["state"][i]) == list(e)
        if kind == "adam":
            assert sd["state"][i]["step"].dtype == e["step"].dtype and sd["state"][i]["step"].device == e["step"].device


# ------------------------------------------------------------------------------------------------
# resume
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["sgd", "adam"])
@pytest.mark.parametrize("ens", ["none", "MCD"])
def test_resumed_run_is_bit_identical(ens, kind):
    """2k steps straight through against k steps, torch.save of the model's and the step's state_dict, a fresh model
    and TrainStep that load both, and k more steps on the same batches, with dropout on: losses at every step,
    parameters, optimizer state, the Adam step count and the dropout step counter are bit-identical."""
    from ta3n_b200.models import VideoModel
    from ta3n_b200.train import Adam, SGDNesterov, TrainStep
    from tests.test_gpu_parity import build_model
    k = 2
    if ens == "MCD":
        from tests.test_mcd_train_step import _gpu_case
        cfg, params, xs0, xt0, labels0, _ = _gpu_case("attn_t4_mu07", dropout=0.5)
        mu, beta = 0.7, [0.75, 0.6, 0.5]
    else:
        cfg, params, xs0, xt0, labels0 = _plain_case(seed=21, dropout=0.5)
        mu, beta = 0.0, BETA
    bs, bt = xs0.shape[0], xt0.shape[0]
    g = torch.Generator().manual_seed(77)
    batches = [(xs0 + 0.1 * torch.randn(xs0.shape, generator=g), xt0 + 0.1 * torch.randn(xt0.shape, generator=g),
                labels0.roll(i)) for i in range(2 * k)]

    def make(state=None):
        model = build_model(cfg, params, train=True)
        if state is not None:
            model.load_state_dict(state)
        opt = Adam(lr=0.003, clip_gradient=5.0) if kind == "adam" else SGDNesterov(lr=0.01, clip_gradient=5.0)
        return model, TrainStep(model, bs, bt, beta, gamma=0.003, mu=mu, optimizer=opt)

    def run(step, batches):
        out = []
        for i, (xs, xt, labels) in enumerate(batches):
            step.set_lr(0.003 / (1 + i))
            out.append(step(xs.pin_memory(), xt.pin_memory(), labels).clone())
        return out

    model_a, step_a = make()
    losses_a = run(step_a, batches)
    model_b, step_b = make()
    losses_b = run(step_b, batches[:k])
    buf = io.BytesIO()
    torch.save({"model": model_b.state_dict(), "step": step_b.state_dict()}, buf)
    buf.seek(0)
    del model_b, step_b
    ck = torch.load(buf)
    model_c, step_c = make(ck["model"])
    step_c.load_state_dict(ck["step"])
    for i, (xs, xt, labels) in enumerate(batches[k:], start=k):
        step_c.set_lr(0.003 / (1 + i))
        losses_b.append(step_c(xs.pin_memory(), xt.pin_memory(), labels).clone())
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(losses_a, losses_b)):
        assert torch.equal(a, b), f"loss of step {i}: {a.item()} vs {b.item()}"
    for (na, pa), (nb, pb) in zip(model_a.named_parameters(), model_c.named_parameters()):
        assert na == nb and torch.equal(pa, pb), na
    for attr in (("exp_avg", "exp_avg_sq", "adam_step") if kind == "adam" else ("momentum_buf",)) + ("step_counter",):
        assert torch.equal(getattr(step_a, attr), getattr(step_c, attr)), attr
    assert step_a.state_dict()["step_counter"] == step_c.state_dict()["step_counter"]


# ------------------------------------------------------------------------------------------------
# the device sampler, and the learning rate of a host running ahead
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["legacy", "phased", "mcd", "legacy_eager"])
def test_adam_step_from_device_sampler_is_bit_identical_to_load(tmp_path, mode):
    """TrainStep+Adam fed by the device sampler against one fed the same batches through load(), over two epochs with
    short last batches: loss, parameters, both moments and the step count equal bit for bit after every step."""
    import copy

    from ta3n_b200 import dataset as D
    from ta3n_b200.train import Adam, TrainStep
    from tests.test_device_sampler import _banks, _gpu_model
    T, batch = 5, (8, 6)
    sets, banks = _banks(tmp_path, T, 2048, (21, None), (9, 14), batch)        # 3 iterations, ends 5 + 2
    model_a = _gpu_model(mode == "mcd")
    model_b = copy.deepcopy(model_a)
    kw = dict(beta=[0.75, 0.75, 0.5], seed=123, mode="phased" if mode == "phased" else "legacy",
              use_graph=mode != "legacy_eager", mu=0.7 if mode == "mcd" else 0.0)
    sampler = D.DevicePairedSampler(banks[0], banks[1], batch, seed=4)
    step_a = TrainStep(model_a, *batch, sampler=sampler, optimizer=Adam(lr=0.003, clip_gradient=5.0), **kw)
    step_b = TrainStep(model_b, *batch, optimizer=Adam(lr=0.003, clip_gradient=5.0), **kw)
    loader = D.PairedFeatureLoader(sets[0], sets[1], batch, seed=4)
    n_step = 0
    for epoch in range(2):
        assert sampler.start_epoch() == len(loader) == 3
        for (xs, ys), (xt, _) in loader:
            if xs.shape[0] < batch[0] or xt.shape[0] < batch[1]:
                step_b.xs.zero_(), step_b.xt.zero_(), step_b.labels.zero_()
            step_b.load(xs, xt, ys)
            loss_b = step_b.run().clone()
            loss_a = step_a.run().clone()
            torch.cuda.synchronize()
            n_step += 1
            assert torch.equal(loss_a, loss_b), (epoch, n_step, loss_a.item(), loss_b.item())
            for attr in ("flat_param", "exp_avg", "exp_avg_sq", "adam_step"):
                assert torch.equal(getattr(step_a, attr), getattr(step_b, attr)), (attr, epoch, n_step)
    assert n_step == 6 and int(step_a.adam_step.item()) == 6


@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_set_lr_keeps_each_value_when_the_host_runs_ahead(kind):
    """set_lr twice while the stream is still busy: each value reaches the stream in order (a copy from a pinned
    buffer that the second call rewrites before the first copy has run would deliver the second value twice)."""
    from ta3n_b200.train import Adam, SGDNesterov, TrainStep
    from tests.test_gpu_parity import build_model
    cfg, params, xs, xt, labels = _plain_case(seed=3)
    opt = Adam(lr=0.5) if kind == "adam" else SGDNesterov(lr=0.5)
    step = TrainStep(build_model(cfg, params, train=True), 12, 7, BETA, optimizer=opt)
    torch.cuda.synchronize()
    seen = []
    torch.cuda._sleep(int(50e-3 * 1.9e9))         # the stream stays busy for ~50 ms while the host enqueues below
    for lr in (0.125, 0.25, 0.0625):
        step.set_lr(lr)
        seen.append(step.lr_dev.clone())
    torch.cuda.synchronize()
    assert [float(t) for t in seen] == [0.125, 0.25, 0.0625]
