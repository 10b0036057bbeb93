"""--optimizer Adam and optimizer checkpoints in torch.optim's format, without a GPU.

The fp64 Adam statement (tests/optim_oracle.py) against torch.optim.Adam; the conversion between TrainStep's flat
optimizer buffers and torch.optim's ``state_dict()`` on a CPU VideoModel (plain and ens_DA='MCD'): it loads into a
stock optimizer, has a stock optimizer's keys, round-trips bit for bit, refuses what the fused update cannot continue,
and never hands out views of the flat buffers; the C ABI's argument checks of the Adam entry; TrainStep's Adam options.
"""
import inspect

import pytest
import torch

from tests import optim_oracle as oo

LR = 0.01


# ------------------------------------------------------------------------------------------------
# the fp64 statement of torch.optim.Adam
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("foreach", [False, None])
def test_oracle_adam_step_matches_torch_optim(foreach):
    """Five steps with weight decay and a learning rate that changes between steps; 'b' never has a gradient and
    'c' only from the third step on (so its step count lags), as with parameters whose .grad is None."""
    g = torch.Generator().manual_seed(3)
    init = {"a": torch.randn(7, 5, generator=g, dtype=torch.float64), "b": torch.randn(3, generator=g, dtype=torch.float64),
            "c": torch.randn(11, generator=g, dtype=torch.float64)}
    ref = {k: torch.nn.Parameter(v.clone()) for k, v in init.items()}
    opt = torch.optim.Adam(ref.values(), lr=LR, betas=(0.8, 0.99), eps=1e-6, weight_decay=3e-2, foreach=foreach)
    params = {k: v.clone() for k, v in init.items()}
    state = {}
    for it in range(5):
        lr = LR / (1 + it)
        for grp in opt.param_groups:
            grp["lr"] = lr
        grads = {"a": torch.randn(7, 5, generator=g, dtype=torch.float64) * (1 + it)}
        if it >= 2:
            grads["c"] = torch.randn(11, generator=g, dtype=torch.float64)
        for k, p in ref.items():
            p.grad = grads[k].clone() if k in grads else None
        opt.step()
        oo.adam_step(params, grads, state, lr, betas=(0.8, 0.99), eps=1e-6, weight_decay=3e-2)
    assert torch.equal(params["b"], init["b"]) and "b" not in state and ref["b"] not in opt.state
    for k in ("a", "c"):
        st = opt.state[ref[k]]
        assert float(st["step"]) == state[k]["step"] == (5 if k == "a" else 3)
        for name, got in (("param", params[k]), ("exp_avg", state[k]["exp_avg"]),
                          ("exp_avg_sq", state[k]["exp_avg_sq"])):
            want = ref[k].detach() if name == "param" else st[name]
            assert torch.allclose(got, want, rtol=1e-14, atol=1e-300), (k, name, (got - want).abs().max())


def test_adam_defaults_are_torch_and_opts():
    from ta3n_b200 import opts
    from ta3n_b200.train import Adam
    sig = inspect.signature(torch.optim.Adam).parameters
    a = Adam(lr=0.1)
    assert a.betas == sig["betas"].default and a.eps == sig["eps"].default
    args = opts.build_parser().parse_args(["classInd.txt", "RGB", "source.txt", "target.txt", "val.txt"])
    assert a.weight_decay == args.weight_decay == 1e-4          # what main.py:86 passes
    assert a.clip_gradient == args.clip_gradient


# ------------------------------------------------------------------------------------------------
# flat buffers <-> torch.optim state_dict on a CPU model
# ------------------------------------------------------------------------------------------------
def _model(ens="none"):
    from ta3n_b200.models import VideoModel
    torch.manual_seed(0)
    return VideoModel(5, "video", "trn-m", "RGB", train_segments=5, val_segments=5, fc_dim=64, ens_DA=ens,
                      verbose=False).train()


def _layout(model, idle=()):
    """Flat size, the per-element update mask (``idle`` path-parameter slots masked out, as TrainStep masks the
    parameters a configuration gives no gradient) and (path param, offset) pairs."""
    from ta3n_b200.train import bucket_layout, step_parameters
    params = step_parameters(model)
    order, offs, n, _ = bucket_layout(params)
    active = torch.ones(n)
    for j in idle:
        active[offs[j]:offs[j] + -(-params[j].numel() // 64) * 64] = 0
    return n, active, [(params[j], offs[j]) for j in order]


def _flat_state(model, keys, active, seed=1):
    """Random flat buffers, zero in the padding and in masked slots (what the kernels leave there)."""
    n, _, slots = _layout(model)
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k in keys:
        buf = torch.zeros(n)
        for p, off in slots:
            if active[off] != 0:
                v = torch.randn(p.numel(), generator=g)
                buf[off:off + p.numel()] = v.abs() if k == "exp_avg_sq" else v
        out[k] = buf
    return out


def _cfg(kind):
    from ta3n_b200.train import Adam, SGDNesterov
    return Adam(lr=LR) if kind == "adam" else SGDNesterov(lr=LR)


def _stock(model, kind, **kw):
    if kind == "adam":
        return torch.optim.Adam(model.parameters(), LR, weight_decay=1e-4, **kw)
    return torch.optim.SGD(model.parameters(), LR, momentum=0.9, weight_decay=1e-4, nesterov=True, **kw)


KEYS = {"adam": ("exp_avg", "exp_avg_sq"), "sgd": ("momentum_buffer",)}
CASES = [("none", ()), ("none", (2, 3, 4, 5)), ("MCD", ())]      # (ens_DA, idle path-parameter slots)


@pytest.mark.parametrize("kind", ["sgd", "adam"])
@pytest.mark.parametrize("ens,idle", CASES)
def test_exported_state_is_a_stock_optimizers(kind, ens, idle):
    from ta3n_b200.train import optimizer_state_from_torch, optimizer_state_to_torch
    model = _model(ens)
    n, active, slots = _layout(model, idle)
    flat = _flat_state(model, KEYS[kind], active)
    cfg = _cfg(kind)
    assert optimizer_state_to_torch(model, cfg, flat, active, step=0)["state"] == {}     # before the first update
    sd = optimizer_state_to_torch(model, cfg, flat, active, step=4)

    # a stock optimizer whose updated parameters (and only those) received gradients
    stock = _stock(model, kind)
    for p in model.parameters():
        p.grad = None
    for p, off in slots:
        if active[off] != 0:
            p.grad = torch.zeros_like(p)
    stock.step()
    want = stock.state_dict()
    assert sd.keys() == want.keys()
    assert sd["param_groups"] == want["param_groups"]
    assert sd["state"].keys() == want["state"].keys()
    for i in want["state"]:
        assert list(sd["state"][i]) == list(want["state"][i])
    index = {id(p): i for i, p in enumerate(model.parameters())}
    if ens == "MCD":
        assert index[id(model.fc_classifier_video_source_2.weight)] in sd["state"]
    if kind == "adam":
        assert all(float(e["step"]) == 4.0 and e["step"].dtype == want["state"][i]["step"].dtype
                   for i, e in sd["state"].items())

    # it loads into a stock optimizer, whose state is then the flat buffers' bit for bit
    fresh = _stock(model, kind)
    fresh.load_state_dict(sd)
    for p, off in slots:
        if active[off] == 0:
            assert p not in fresh.state
            continue
        for k in KEYS[kind]:
            assert torch.equal(fresh.state[p][k].reshape(-1), flat[k][off:off + p.numel()])

    # the exported tensors own their storage: no view of the flat buffers
    flat_ptrs = {t.untyped_storage().data_ptr() for t in flat.values()}
    for e in sd["state"].values():
        for k in KEYS[kind]:
            t = e[k]
            assert t.untyped_storage().data_ptr() not in flat_ptrs
            assert t.untyped_storage().nbytes() == t.numel() * 4

    # flat -> dict -> flat is bit-identical, padding and masked slots included
    back = {k: torch.full_like(v, 7.0) for k, v in flat.items()}
    lr, step = optimizer_state_from_torch(model, cfg, sd, back, active)
    assert lr == LR and step == (4 if kind == "adam" else 1)
    for k in KEYS[kind]:
        assert torch.equal(back[k], flat[k])
    # a dict the stock optimizer saves after the same point loads as well
    lr, step = optimizer_state_from_torch(model, cfg, fresh.state_dict(), back, active)
    for k in KEYS[kind]:
        assert torch.equal(back[k], flat[k])


@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_empty_state_loads_as_zero_state(kind):
    from ta3n_b200.train import optimizer_state_from_torch
    model = _model()
    _, active, _ = _layout(model)
    flat = _flat_state(model, KEYS[kind], active)
    lr, step = optimizer_state_from_torch(model, _cfg(kind), _stock(model, kind, ).state_dict(), flat, active)
    assert (lr, step) == (LR, 0)
    assert all(not v.any() for v in flat.values())


def _stepped(model, active, cls, **kw):
    """state_dict of a stock ``cls`` over model.parameters() after one step in which the updated parameters had a
    gradient."""
    _, _, slots = _layout(model)
    g = torch.Generator().manual_seed(9)
    for p in model.parameters():
        p.grad = None
    for p, off in slots:
        if active[off] != 0:
            p.grad = torch.randn(p.shape, generator=g)
    opt = cls(model.parameters(), LR, **kw)
    with torch.no_grad():
        saved = [p.clone() for p in model.parameters()]
        opt.step()
        for p, v in zip(model.parameters(), saved):
            p.copy_(v)
    return opt.state_dict()


# optimizers whose state_dict shares names with SGD's or Adam's (momentum_buffer; betas, step, exp_avg, exp_avg_sq)
OTHER_OPTIMIZERS = {
    "RMSprop": (torch.optim.RMSprop, dict(momentum=0.9, weight_decay=1e-4)),
    "NAdam": (torch.optim.NAdam, dict(weight_decay=1e-4)),
    "RAdam": (torch.optim.RAdam, dict(weight_decay=1e-4)),
    "Adamax": (torch.optim.Adamax, dict(weight_decay=1e-4)),
    "Adagrad": (torch.optim.Adagrad, dict(weight_decay=1e-4)),
    "AdamW": (torch.optim.AdamW, dict(weight_decay=1e-4)),
    "Adam amsgrad": (torch.optim.Adam, dict(weight_decay=1e-4, amsgrad=True)),
    "SGD plain momentum": (torch.optim.SGD, dict(momentum=0.9, weight_decay=1e-4)),
}


def _refusals(model, kind, sd, idle_index, active):
    """(what, state_dict) pairs the fused update cannot continue."""
    import copy
    out = []

    def edit(what, fn):
        d = copy.deepcopy(sd)
        fn(d)
        out.append((what, d))

    other = torch.optim.SGD(model.parameters(), LR, momentum=0.9, nesterov=True) if kind == "adam" else \
        torch.optim.Adam(model.parameters(), LR)
    out.append(("other optimizer type", other.state_dict()))
    for name, (cls, kw) in OTHER_OPTIMIZERS.items():
        out.append((name, _stepped(model, active, cls, **kw)))
    out.append(("the other of SGD / Adam, stepped", _stepped(model, active, torch.optim.SGD, momentum=0.9,
                                                              weight_decay=1e-4, nesterov=True) if kind == "adam" else
                _stepped(model, active, torch.optim.Adam, weight_decay=1e-4)))
    edit("a key of another optimizer", lambda d: d["param_groups"][0].update(momentum_decay=4e-3))
    edit("a key of this optimizer missing",
         lambda d: d["param_groups"][0].pop("amsgrad" if kind == "adam" else "nesterov"))
    edit("a state entry of another name", lambda d: d["state"][next(iter(d["state"]))].update(
        square_avg=torch.zeros_like(d["state"][next(iter(d["state"]))][KEYS[kind][0]])))
    params = list(model.parameters())
    two = type(_stock(model, kind))([{"params": params[:5]}, {"params": params[5:]}], LR)
    out.append(("two param groups", two.state_dict()))
    edit("a parameter count that differs", lambda d: d["param_groups"][0].update(params=d["param_groups"][0]["params"][:-1]))
    if kind == "adam":
        edit("betas", lambda d: d["param_groups"][0].update(betas=(0.8, 0.999)))
        edit("eps", lambda d: d["param_groups"][0].update(eps=1e-6))
        edit("weight decay", lambda d: d["param_groups"][0].update(weight_decay=0.0))
        edit("amsgrad", lambda d: d["param_groups"][0].update(amsgrad=True))
        edit("maximize", lambda d: d["param_groups"][0].update(maximize=True))
        edit("decoupled weight decay", lambda d: d["param_groups"][0].update(decoupled_weight_decay=True))
        out.append(("AdamW", torch.optim.AdamW(model.parameters(), LR, weight_decay=1e-4).state_dict()))
        first = next(iter(sd["state"]))
        edit("steps that differ", lambda d: d["state"][first].update(step=torch.tensor(2.0)))
        edit("state missing for an updated parameter", lambda d: d["state"].pop(first))
        edit("a step that is not a positive integer", lambda d: [e.update(step=torch.tensor(2.5))
                                                               for e in d["state"].values()])
    else:
        edit("momentum", lambda d: d["param_groups"][0].update(momentum=0.8))
        edit("weight decay", lambda d: d["param_groups"][0].update(weight_decay=1e-3))
        edit("dampening", lambda d: d["param_groups"][0].update(dampening=0.1))
        edit("nesterov", lambda d: d["param_groups"][0].update(nesterov=False))
        edit("maximize", lambda d: d["param_groups"][0].update(maximize=True))
    some = next(iter(sd["state"].values()))
    edit("state for a parameter the update never touches", lambda d: d["state"].update({idle_index: some}))
    edit("a state tensor of the wrong shape",
         lambda d: d["state"][next(iter(d["state"]))].update({KEYS[kind][0]: torch.zeros(3)}))
    return out


@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_refusals_raise_value_error_and_write_nothing(kind):
    from ta3n_b200.train import optimizer_state_from_torch, optimizer_state_to_torch
    model = _model()
    _, active, _ = _layout(model, idle=(2, 3, 4, 5))         # frame discriminator idle
    flat = _flat_state(model, KEYS[kind], active)
    sd = optimizer_state_to_torch(model, _cfg(kind), flat, active, step=3)
    idle_index = [i for i, p in enumerate(model.parameters()) if p is model.fc_feature_domain.weight][0]
    assert idle_index not in sd["state"]
    keep = {k: v.clone() for k, v in flat.items()}
    cases = _refusals(model, kind, sd, idle_index, active)
    assert len(cases) >= (27 if kind == "adam" else 22)
    for what, bad in cases:
        with pytest.raises(ValueError):
            optimizer_state_from_torch(model, _cfg(kind), bad, flat, active)
            pytest.fail(f"accepted: {what}")
        assert all(torch.equal(flat[k], keep[k]) for k in flat), what


@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_a_group_without_the_switches_of_newer_torch_loads(kind):
    """A param group written by an older torch lacks switches added since (maximize, foreach, capturable,
    differentiable, fused, decoupled_weight_decay); they were off then, and such a dict still loads."""
    from ta3n_b200.train import optimizer_state_from_torch, optimizer_state_to_torch
    model = _model()
    _, active, _ = _layout(model)
    flat = _flat_state(model, KEYS[kind], active)
    sd = optimizer_state_to_torch(model, _cfg(kind), flat, active, step=2)
    for k in ("maximize", "foreach", "capturable", "differentiable", "fused", "decoupled_weight_decay"):
        sd["param_groups"][0].pop(k, None)
    back = {k: torch.zeros_like(v) for k, v in flat.items()}
    assert optimizer_state_from_torch(model, _cfg(kind), sd, back, active) == (LR, 2 if kind == "adam" else 1)
    assert all(torch.equal(back[k], flat[k]) for k in flat)


# ------------------------------------------------------------------------------------------------
# TrainStep options and the C ABI's argument checks (host only)
# ------------------------------------------------------------------------------------------------
def test_train_step_refuses_bad_adam_configurations_before_the_device():
    from ta3n_b200.train import Adam, TrainStep
    m = _model()
    for bad in (Adam(lr=0.1, betas=(1.0, 0.999)), Adam(lr=0.1, betas=(0.9, -0.1)), Adam(lr=0.1, eps=0.0),
                Adam(lr=0.1, weight_decay=-1e-4)):
        with pytest.raises(ValueError):
            TrainStep(m, 4, 4, beta=[0.75, 0.75, 0.5], optimizer=bad)
    with pytest.raises(TypeError):
        TrainStep(m, 4, 4, beta=[0.75, 0.75, 0.5], optimizer=torch.optim.Adam(m.parameters()))


def test_adam_entry_validates_arguments_without_a_gpu():
    from ta3n_b200 import build
    build.build()
    from ta3n_b200 import _lib
    lib = _lib.load()
    ws = lib.ta3n_adam_workspace_bytes()
    assert ws >= 296 * 4 + 4

    def call(p=16, g=32, m=48, v=64, n=10, lr=80, step=96, b1=0.9, b2=0.999, eps=1e-8, wd=1e-4, clip=0.0, w=128,
             wb=ws, active=None):
        return lib.ta3n_adam_step_masked(p, g, m, v, n, lr, step, b1, b2, eps, wd, clip, w, wb, None, active, None)

    # every call below fails a host-side check before anything is launched
    for kw, msg in ((dict(p=None), b"bad arguments"), (dict(step=None), b"bad arguments"), (dict(n=0), b"bad arguments"),
                    (dict(m=52), b"16-byte aligned"), (dict(active=20), b"16-byte aligned"),
                    (dict(b1=1.0), b"betas"), (dict(b2=-0.5), b"betas"), (dict(b1=float("nan")), b"betas"),
                    (dict(eps=0.0), b"eps"), (dict(wd=-1.0), b"eps"), (dict(w=None), b"workspace"),
                    (dict(wb=ws - 1), b"workspace")):
        assert call(**kw) == 1, kw
        assert msg in lib.ta3n_last_error(), (kw, lib.ta3n_last_error())
