"""TrainStep(pretrain_source=True): the source-only pre-training update of main.py:388-414 ahead of each adaptation
iteration, in the same captured step.

CPU: the oracle (oracle/pretrain_oracle.py) against the reference's iterations (tests/golden/pretrain_golden.npz, and
the live reference where it is present), the options TrainStep refuses with it, and the optimizer state rules (Adam's
2k / k step counts).
GPU: one iteration against the fp64 oracle on the fp32, tf32x3 and tf32 engines, with the ReLU pattern of every pass
pinned, dropout off and on, over the attention variants, add_fc 2, MCD, DAN, target entropy, short batches, SGD and
Adam (Adam on fp32); three
iterations against the stock autograd loop with torch.optim; bit-identical eager / graph / reruns, resume and device
sampler; the meters; the launches the option adds.
"""
import copy
import itertools
import os

import pytest
import torch

from oracle import add_fc_oracle as afo
from oracle import dis_oracle as dor
from oracle import mcd_oracle as mcd
from oracle import pretrain_oracle as pto
from oracle import ref_shims
from oracle import ta3n_oracle as orc
from oracle import target_entropy_oracle as teo
from tests.golden_util import assert_close

gpu = pytest.mark.gpu
BETA = (0.75, 0.6, 0.5)


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------
def _cpu_model(**kw):
    from ta3n_b200.models import VideoModel
    args = dict(train_segments=5, val_segments=5, fc_dim=64, verbose=False)
    args.update(kw)
    return VideoModel(5, "video", "trn-m", "RGB", **args).train()


@pytest.mark.parametrize("ens", ["none", "MCD"])
def test_train_step_refusals(ens):
    from ta3n_b200 import Ta3nError
    from ta3n_b200.train import Adam, SGDNesterov, TrainStep
    m = _cpu_model(ens_DA=ens)
    kw = dict(pretrain_source=True, optimizer=SGDNesterov(lr=0.01))
    with pytest.raises(NotImplementedError, match="legacy"):
        TrainStep(m, 4, 4, beta=BETA, mode="phased", **kw)
    with pytest.raises(NotImplementedError, match="step program"):
        TrainStep(m, 4, 4, beta=BETA, class_weight=torch.ones(5), **kw)
    with pytest.raises(NotImplementedError, match="step program"):
        TrainStep(m, 4, 4, beta=BETA, domain_weight=(1.0, 0.5), **kw)
    with pytest.raises(NotImplementedError, match="step program"):
        TrainStep(m, 4, 4, beta=[-1.0, 0.75, 0.5], **kw)
    with pytest.raises(ValueError, match="optimizer"):
        TrainStep(m, 4, 4, beta=BETA, pretrain_source=True)
    # the accepted configurations pass every check and stop at the device
    for opt in (SGDNesterov(lr=0.01), Adam(lr=1e-3)):
        with pytest.raises(Ta3nError, match="CUDA"):
            TrainStep(m, 4, 4, beta=BETA, pretrain_source=True, optimizer=opt)


def _pretrain_layout(model, idle=()):
    """The update mask and the pre-training mask of the CPU model's flat buffers; P from the oracle's gradients."""
    from tests.test_optimizer_state import _layout
    from ta3n_b200.train import bucket_layout, step_parameters
    n, active, slots = _layout(model, idle)
    cfg = orc.PathConfig(num_class=5, num_segments=5, fc_dim=64, use_attn=model.use_attn,
                         use_attn_frame=model.use_attn_frame, ens_DA=model.ens_DA)
    params = {k: v.detach().double() for k, v in model.state_dict().items()}
    xs = torch.randn(3, 5, orc.FEATURE_DIM, dtype=torch.float64)
    _, grads = pto.pretrain_step(params, xs, torch.arange(3), BETA, cfg)
    reached = {id(p) for name, p in model.named_parameters() if grads.get(name) is not None}
    sp = step_parameters(model)
    _, offs, _, _ = bucket_layout(sp)
    pre = torch.zeros(n)
    for p in sp:
        if id(p) in reached:
            j = [id(q) for q in sp].index(id(p))
            pre[offs[j]:offs[j] + -(-p.numel() // 64) * 64] = 1
    return active, pre, reached


def _adaptation_reached(model, place_adv, add_loss_DA):
    """Names of the parameters that get a gradient in the fp64 oracle's adaptation loss (MCD: both passes)."""
    cfg = orc.PathConfig(num_class=5, num_segments=5, fc_dim=64, use_attn=model.use_attn,
                         use_attn_frame=model.use_attn_frame, ens_DA=model.ens_DA)
    params = {k: v.detach().double() for k, v in model.state_dict().items()}
    names = orc.used_param_names(params)
    live = dict(params, **{k: params[k].clone().requires_grad_(True) for k in names})
    xs, xt = (torch.randn(3, 5, orc.FEATURE_DIM, dtype=torch.float64) for _ in range(2))
    labels = torch.arange(3)
    attn = model.use_attn if add_loss_DA == "attentive_entropy" else "none"
    o1 = orc.forward(live, xs, xt, BETA, 0.0, cfg)
    if model.ens_DA == "MCD":
        o2 = mcd.pass2_target(live, xt, BETA, 0.0, cfg)
        loss = mcd.mcd_loss(o1, o1[2], (o2[1], o2[2]), labels, 0.003, attn, place_adv)
    else:
        loss = orc.compose_loss(o1, labels, 0.003, place_adv=place_adv, use_attn=attn)
    if add_loss_DA == "target_entropy":
        loss = loss + 0.003 * teo.target_entropy(o1[6])
    grads = torch.autograd.grad(loss, [live[k] for k in names], allow_unused=True)
    return {k for k, g in zip(names, grads) if g is not None}


@pytest.mark.parametrize("attn,attn_frame", [("TransAttn", "none"), ("none", "none"), ("TransAttn", "TransAttn")])
@pytest.mark.parametrize("ens", ["none", "MCD"])
def test_update_set_and_p_are_what_the_oracle_losses_reach(attn, attn_frame, ens):
    """The slots the fused update keeps (all but ``idle_slots``) are the parameters the fp64 oracle's adaptation loss
    gives a gradient, for every place_adv and add_loss_DA TrainStep accepts; ``pretrain_slots`` (P) are those its
    source-only loss gives one."""
    from ta3n_b200.train import idle_slots, pretrain_slots, step_parameters
    m = _cpu_model(use_attn=attn, use_attn_frame=attn_frame, ens_DA=ens)
    sp = step_parameters(m)
    name = {id(p): k for k, p in m.named_parameters()}
    slots = lambda names: {j for j, p in enumerate(sp) if name[id(p)] in names}     # noqa: E731
    for place_adv in itertools.product("YN", repeat=3):
        for add_loss_DA in ("attentive_entropy", "none", "target_entropy"):
            entropy = add_loss_DA == "attentive_entropy" and attn != "none"
            if entropy and place_adv[:2] != ("Y", "Y"):
                continue        # refused: the attentive entropy reads the video level
            flags = (place_adv[0] == "Y") | (place_adv[1] == "Y") << 1 | (place_adv[2] == "Y") << 2 | entropy << 3
            kept = set(range(len(sp))) - set(idle_slots(m, flags))
            assert kept == slots(_adaptation_reached(m, place_adv, add_loss_DA)), (place_adv, add_loss_DA)
    cfg = orc.PathConfig(num_class=5, num_segments=5, fc_dim=64, use_attn=attn, use_attn_frame=attn_frame, ens_DA=ens)
    params = {k: v.detach().double() for k, v in m.state_dict().items()}
    xs = torch.randn(3, 5, orc.FEATURE_DIM, dtype=torch.float64)
    _, grads = pto.pretrain_step(params, xs, torch.arange(3), BETA, cfg)
    assert set(pretrain_slots(m)) == slots({k for k, g in grads.items() if g is not None})


@pytest.mark.parametrize("attn,ens", [("TransAttn", "none"), ("none", "none"), ("TransAttn", "MCD")])
def test_adam_state_round_trip_and_stock_checkpoint(attn, ens):
    """The exported state holds step 2k for P and k for the rest; a stock torch.optim.Adam state with those counts
    (a reference run with --pretrain_source) loads and gives k back, and loads into a stock optimizer."""
    from tests.test_optimizer_state import _flat_state, _stock
    from ta3n_b200.train import Adam, optimizer_state_from_torch, optimizer_state_to_torch
    model = _cpu_model(use_attn=attn, ens_DA=ens)
    idle = (2, 3, 4, 5) if attn == "none" else ()
    active, pre, reached = _pretrain_layout(model, idle)
    assert pre.sum() > 0 and torch.all(pre <= active)
    cfg = Adam(lr=1e-3)
    flat = _flat_state(model, ("exp_avg", "exp_avg_sq"), active)
    sd = optimizer_state_to_torch(model, cfg, flat, active, step=3, pretrain=pre)
    params = list(model.parameters())
    for i, entry in sd["state"].items():
        assert float(entry["step"]) == (6.0 if id(params[i]) in reached else 3.0)
    stock = _stock(model, "adam")
    stock.load_state_dict(copy.deepcopy(sd))
    back = {k: torch.zeros_like(v) for k, v in flat.items()}
    lr, step = optimizer_state_from_torch(model, cfg, stock.state_dict(), back, active, pretrain=pre)
    assert step == 3 and lr == stock.param_groups[0]["lr"]
    for k in flat:
        assert torch.equal(back[k], flat[k])


def test_adam_step_counts_are_checked():
    from tests.test_optimizer_state import _flat_state
    from ta3n_b200.train import Adam, optimizer_state_from_torch, optimizer_state_to_torch
    model = _cpu_model()
    active, pre, reached = _pretrain_layout(model)
    cfg = Adam(lr=1e-3)
    flat = _flat_state(model, ("exp_avg", "exp_avg_sq"), active)
    paired = optimizer_state_to_torch(model, cfg, flat, active, step=2, pretrain=pre)
    equal = optimizer_state_to_torch(model, cfg, flat, active, step=2)
    back = {k: torch.zeros_like(v) for k, v in flat.items()}
    # the default keeps refusing unequal counts; with the mask, equal counts are refused
    with pytest.raises(ValueError, match="equal steps"):
        optimizer_state_from_torch(model, cfg, paired, back, active)
    with pytest.raises(ValueError, match="pre-training"):
        optimizer_state_from_torch(model, cfg, equal, back, active, pretrain=pre)
    odd = copy.deepcopy(paired)
    params = list(model.parameters())
    i = next(i for i in odd["state"] if id(params[i]) in reached)
    odd["state"][i]["step"] = torch.tensor(3.0)
    with pytest.raises(ValueError):
        optimizer_state_from_torch(model, cfg, odd, back, active, pretrain=pre)
    assert optimizer_state_from_torch(model, cfg, paired, back, active, pretrain=pre)[1] == 2


# ------------------------------------------------------------------------------------------------
# CPU: the oracle against the reference's iterations (tests/golden/pretrain_golden.npz)
# ------------------------------------------------------------------------------------------------
def _golden():
    import json
    import numpy as np
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pretrain_golden.npz"))
    return z, json.loads(bytes(z["meta_json"]).decode())


def _real_masks(c, m, dom_rows):
    """The keep masks of the real rows, for the given domains: {domain: rows}."""
    T = c["T"]
    out = {}
    for k, v in m.items():
        dom = k.rsplit("_", 1)[1]
        if dom in dom_rows:
            out[k] = v[:dom_rows[dom] * (T if k.startswith("i") else 1)]
    return out


def _oracle_run(c, dtype=torch.float64):
    """The oracle's records of the golden case, in the generator's format (``gen_golden_pretrain.run_reference``)."""
    from oracle import gen_golden_pretrain as gen
    from tests.optim_oracle import adam_step
    cfg = gen.case_config(c)
    p = {k: v.to(dtype) for k, v in gen.case_params(c).items()}
    xs, xt, labels = gen.case_inputs(c)
    ns, nt = c["ns"], c["nt"]
    xs, xt, labels = xs[:ns].to(dtype), xt[:nt].to(dtype), labels[:ns]
    state, bufs = {}, {}
    if c["opt"] == "adam":
        update = lambda q, g: adam_step(q, g, state, gen.LR_ADAM)                          # noqa: E731
    else:
        update = lambda q, g: orc.sgd_nesterov_step(q, g, bufs, gen.LR_SGD, 0.9, 1e-4)     # noqa: E731
    runs = []
    for it in range(gen.ITERATIONS):
        rec = {}
        m_pre = _real_masks(c, gen.case_masks(c, it, 0), {"source": ns})
        m = _real_masks(c, gen.case_masks(c, it, 1), {"source": ns, "target": nt})
        m2 = _real_masks(c, gen.case_masks(c, it, 2), {"target": nt}) if c["ens"] == "MCD" else None
        loss, g1 = pto.pretrain_step(p, xs, labels, gen.BETA, cfg, c["add_fc"], masks=m_pre)
        rec["with_grad_pre"] = sorted(k for k, g in g1.items() if g is not None)
        rec["loss_pre"] = loss.item()
        pto.apply_update(p, g1, update, gen.CLIP)
        rec["params_pre"] = {k: v.clone() for k, v in p.items()}
        if c["extra"] == "target_entropy":
            loss, _, g2 = teo.entropy_train_step(p, xs, xt, labels, gen.BETA, cfg, gen.GAMMA, masks=m, mu=c["mu"],
                                                 masks2=m2)
        elif c["extra"] == "DAN":
            loss, _, g2 = dor.dis_train_step(p, xs, xt, labels, gen.BETA, cfg, "DAN", gen.ALPHA, gen.PLACE_DIS,
                                             c["add_fc"], gen.GAMMA, masks=m, mu=c["mu"], masks2=m2)
        elif c["ens"] == "MCD":
            loss, _, _, g2 = mcd.mcd_train_step(p, xs, xt, labels, gen.BETA, c["mu"], cfg, gen.GAMMA, masks=m,
                                                masks2=m2)
        else:
            loss, _, g2 = afo.train_step(p, xs, xt, labels, gen.BETA, cfg, c["add_fc"], gen.GAMMA, masks=m)
        rec["loss"] = loss.item()
        pto.apply_update(p, g2, update, gen.CLIP)
        rec["params"] = {k: v.clone() for k, v in p.items()}
        if c["opt"] == "adam":
            rec["state"] = {k: {"step": float(st["step"]), "exp_avg": st["exp_avg"].clone(),
                                "exp_avg_sq": st["exp_avg_sq"].clone()} for k, st in state.items()}
        else:
            rec["state"] = {k: {"momentum_buffer": b.clone()} for k, b in bufs.items()}
        runs.append(rec)
    return runs


def _unpack(vec, layout):
    out = {}
    for name, off, n_head, n_sample in layout:
        head = torch.from_numpy(vec[off:off + n_head])
        out[name] = (head, torch.from_numpy(vec[off + n_head:off + n_head + n_sample]) if n_sample else None)
    return out


def _check_stored(got, stored, init, tol, what, noise):
    """``got`` against a packed tensor: a whole one by its change from ``init``; a large one by its sum and by the
    change of its strided sample."""
    from oracle import gen_golden_pretrain as gen
    head, sample = stored
    got = got.detach().double().reshape(-1)
    init = init.double().reshape(-1) if init is not None else torch.zeros_like(got)
    if sample is None:
        assert_close(got - init, head - init, tol, what, noise=noise)
        return
    assert abs(got.norm().item() - head[1].item()) <= tol * head[1].item() + 8 * noise, what
    assert_close((got - init)[::gen.STRIDE], sample - init.float().double()[::gen.STRIDE], tol * 4, what + " (sample)",
                 noise=noise)


@pytest.mark.parametrize("case", ["attn", "noattn", "attnframe_t7", "add_fc2", "mcd_mu07", "dan", "entropy", "short",
                                  "adam"])
def test_oracle_equals_golden(case):
    """The oracle's iterations against the reference's main.py:388-583 (tests/golden/pretrain_golden.npz): both losses,
    the parameters with a gradient after the pre-training backward (P), the parameters after each update, and the
    optimizer state with Adam's per-parameter step counts (2k for P, k for the rest)."""
    from oracle import gen_golden_pretrain as gen
    z, meta = _golden()
    c = gen.case(case)
    init = gen.case_params(c)
    runs = _oracle_run(c)
    for it, rec in enumerate(runs):
        k = f"{case}/{it}/"
        noise = meta[k + "noise"]
        assert rec["with_grad_pre"] == sorted(meta[k + "with_grad_pre"])
        assert not any(n.startswith("fc_feature_domain_video") or n.startswith("fc_classifier_domain_video")
                       for n in rec["with_grad_pre"])
        for key in ("loss_pre", "loss"):
            assert_close(torch.tensor(rec[key]), torch.tensor(meta[k + key]), 1e-5, f"{k}{key}", noise=noise[key])
        for part in ("params_pre", "params"):
            stored = _unpack(z[k + part], meta[k + part + "/layout"])
            assert set(stored) <= set(init) and len(stored) == len(meta[case + "/param_order"])
            for n, t in stored.items():
                _check_stored(rec[part][n], t, init[n], 2e-4, f"{k}{part}/{n}",
                              max(noise[part + "/" + n], 1e-9))
        stored = _unpack(z[k + "state"], meta[k + "state/layout"])
        assert sorted(rec["state"]) == sorted(meta[k + "state_names"])
        if c["opt"] == "adam":
            want = {n: (2 * (it + 1) if n in rec["with_grad_pre"] else it + 1) for n in rec["state"]}
            assert {n: st["step"] for n, st in rec["state"].items()} == meta[k + "steps"] == want
        for key, t in stored.items():
            n, sk = key.rsplit("/", 1)
            _check_stored(rec["state"][n][sk], t, None, 2e-4 if sk != "exp_avg_sq" else 5e-4, f"{k}state/{key}",
                          max(noise["state/" + key], 1e-9))


@pytest.mark.skipif(not ref_shims.available(), reason="needs the reference tree")
@pytest.mark.parametrize("case", ["attn", "noattn", "mcd_mu07", "adam"])
def test_oracle_equals_live_reference(case):
    from oracle import gen_golden_pretrain as gen
    c = gen.case(case)
    ref, _ = gen.run_reference(c, torch.float64)
    mine = _oracle_run(c)
    for it, (r, o) in enumerate(zip(ref, mine)):
        assert sorted(r["with_grad_pre"]) == o["with_grad_pre"]
        assert o["loss_pre"] == pytest.approx(r["loss_pre"], rel=1e-9)
        assert o["loss"] == pytest.approx(r["loss"], rel=1e-9)
        for part in ("params_pre", "params"):
            for n, t in r[part].items():
                assert_close(o[part][n], t, 1e-9, f"{it} {part}/{n}", noise=1e-12)
        for n, st in r["state"].items():
            for sk, v in st.items():
                if sk == "step":
                    assert o["state"][n][sk] == float(v)
                else:
                    assert_close(o["state"][n][sk], v, 1e-8, f"{it} state/{n}/{sk}", noise=1e-12)


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------
def _dev():
    return torch.device("cuda:0")


def _model(T=5, C=7, drop=0.0, attn="TransAttn", attn_frame="none", ens="none", add_fc=1, seed=3):
    from ta3n_b200.models import VideoModel
    torch.manual_seed(seed)
    m = VideoModel(C, "video", "trn-m", "RGB", train_segments=T, val_segments=T, fc_dim=256, dropout_i=drop,
                   dropout_v=drop, partial_bn=False, use_attn=attn, use_attn_frame=attn_frame, ens_DA=ens,
                   add_fc=add_fc, verbose=False)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for _, v in sorted(m.named_parameters()):
            if v.dim() > 1:
                v.add_(0.02 * torch.randn(v.shape, generator=g))
    return m.to(_dev()).train()


def _inputs(bs, bt, T, seed=9):
    g = torch.Generator().manual_seed(seed)
    xs = torch.randn(bs, T, orc.FEATURE_DIM, generator=g)
    xt = torch.randn(bt, T, orc.FEATURE_DIM, generator=g) * 1.2 - 0.3
    return xs, xt, torch.arange(bs) % 7


CASES = {
    # name: (attn, attn_frame, ens, mu, add_fc, drop, (Bs, Bt), (ns, nt), extra, opt)
    "attn": ("TransAttn", "none", "none", 0.0, 1, 0.0, (10, 7), (10, 7), None, "sgd"),
    "attn_drop": ("TransAttn", "none", "none", 0.0, 1, 0.5, (10, 7), (10, 7), None, "sgd"),
    "none_drop": ("none", "none", "none", 0.0, 1, 0.5, (8, 9), (8, 9), None, "sgd"),
    "frame_attn_drop": ("TransAttn", "TransAttn", "none", 0.0, 1, 0.5, (7, 9), (7, 9), None, "sgd"),
    "add_fc2_drop": ("TransAttn", "none", "none", 0.0, 2, 0.5, (8, 6), (8, 6), None, "sgd"),
    "mcd_mu0": ("TransAttn", "none", "MCD", 0.0, 1, 0.0, (8, 6), (8, 6), None, "sgd"),
    "mcd_mu07_drop": ("TransAttn", "none", "MCD", 0.7, 1, 0.5, (8, 6), (8, 6), None, "sgd"),
    "dan_drop": ("TransAttn", "none", "none", 0.0, 1, 0.5, (10, 7), (10, 7), "DAN", "sgd"),
    "entropy_drop": ("TransAttn", "none", "none", 0.0, 1, 0.5, (10, 7), (10, 7), "target_entropy", "sgd"),
    "short_drop": ("TransAttn", "none", "none", 0.0, 1, 0.5, (10, 7), (6, 4), None, "sgd"),
    "adam": ("TransAttn", "none", "none", 0.0, 1, 0.0, (10, 7), (10, 7), None, "adam"),
    "adam_none_drop": ("none", "none", "none", 0.0, 1, 0.5, (8, 9), (8, 9), None, "adam"),
}
LR, CLIP, GAMMA, ALPHA = 0.01, 0.5, 0.3, 0.7


CASE_T = {"frame_attn_drop": 7}      # frames per video (default 5)


@pytest.fixture(params=["fp32", "tf32x3", "tf32"])
def engine(request):
    import ta3n_b200
    ta3n_b200.set_gemm_engine(request.param)
    yield request.param
    ta3n_b200.set_gemm_engine("tf32x3")


def _updater(kind):
    """``update(params, grads)`` of the fused optimizer's torch.optim counterpart; per-parameter Adam steps."""
    if kind == "sgd":
        bufs = {}
        return lambda p, g: orc.sgd_nesterov_step(p, g, bufs, LR, 0.9, 1e-4)
    from tests.optim_oracle import adam_step
    state = {}
    return lambda p, g: adam_step(p, g, state, LR * 0.1)


def _adaptation(case, cfg, p, xs, xt, labels, masks, masks2, gates, gates2):
    attn, attn_frame, ens, mu, add_fc, drop, _, _, extra, _ = CASES[case]
    train = drop > 0
    if extra == "target_entropy":
        loss, _, g = teo.entropy_train_step(p, xs, xt, labels, BETA, cfg, GAMMA, train=train, masks=masks, mu=mu,
                                            masks2=masks2, gates=gates, gates2=gates2)
    elif extra == "DAN":
        loss, _, g = dor.dis_train_step(p, xs, xt, labels, BETA, cfg, "DAN", ALPHA, gamma=GAMMA, train=train,
                                        masks=masks, mu=mu, masks2=masks2, gates=gates, gates2=gates2)
    elif ens == "MCD":
        loss, _, _, g = mcd.mcd_train_step(p, xs, xt, labels, BETA, mu, cfg, GAMMA, masks=masks, masks2=masks2,
                                           gates=gates, gates2=gates2)
    else:
        loss, _, g = afo.train_step(p, xs, xt, labels, BETA, cfg, add_fc, GAMMA, train=train, masks=masks, gates=gates)
    return loss, g


def _pinned(pool, add_fc, rows_f, rows_v, masks, plain, frame_disc, video_disc, n_f):
    """The pass's realised ReLU pattern in the oracle's gate format (every shared layer's under add_fc) and its flips
    against the fp64 pattern ``plain``.  ``masks``: the pass's keep masks in domain order (None: no dropout)."""
    from tests.pinned_pattern import realised_gates
    F_ = plain["shared" if add_fc == 1 else f"shared{add_fc}"].shape[1]

    def kept(k):
        parts = [v for key, v in (masks or {}).items() if key.startswith(k + "_")]
        return torch.cat(parts).bool() if parts else torch.ones(n_f, F_, dtype=torch.bool)
    top = "shared" if add_fc == 1 else f"shared{add_fc}"
    top_mask = "i" if add_fc == 1 else f"i{add_fc}"
    gates, flips, total = realised_gates(pool, rows_f, rows_v, kept(top_mask), {**plain, "shared": plain[top]},
                                         frame_disc, video_disc)
    if add_fc > 1:
        gates[top] = gates.pop("shared")
        for layer in range(1, add_fc):
            k, mk = ("shared" if layer == 1 else f"shared{layer}"), ("i" if layer == 1 else f"i{layer}")
            g = torch.where(kept(mk), rows_f(pool[f"feat_{layer}"]) > 0, plain[k])
            flips += ((g != plain[k]) & kept(mk)).sum().item()
            total += kept(mk).sum().item()
            gates[k] = g
    return gates, flips, total


def _oracle_iteration(case, cfg, params, xs, xt, labels, key, step, engine):
    """The fp64 and fp32 oracle iterations on the ReLU patterns the step realised in each pass; (fp64 results, fp32
    results, flips, units counted)."""
    attn, attn_frame, ens, mu, add_fc, drop, (Bs, Bt), (ns, nt), extra, kind = CASES[case]
    T = cfg.num_segments
    masks = masks2 = masks_pre = None
    if drop > 0:
        masks = afo.train_step_masks(key, Bs, Bt, T, cfg.shared_dim, cfg.video_dim, drop, drop, add_fc, ns=ns, nt=nt)
        masks_pre = pto.pretrain_masks(key, Bs, T, cfg.shared_dim, cfg.video_dim, drop, drop, add_fc, ns=ns)
        if ens == "MCD":
            masks2 = mcd.train_step_pass2_masks(key, Bt, T, cfg.shared_dim, cfg.video_dim, drop, drop, nt=nt)
    frames = lambda t: torch.cat([t[:ns * T], t[Bs * T:Bs * T + nt * T]]).cpu()    # noqa: E731
    videos = lambda t: torch.cat([t[:ns], t[Bs:Bs + nt]]).cpu()                    # noqa: E731
    empty = lambda m: None if m is None else {**m, **{k.replace("_source", "_target"): v[:0]     # noqa: E731
                                                       for k, v in m.items()}}
    x64, t64 = xs.double(), xt.double()
    p = {k: v.double() if v.dtype.is_floating_point else v for k, v in params.items()}
    # the pre-training pass: its pattern on the fp64 weights before the update
    plain = afo.activation_pattern(p, x64, x64[:0], BETA, cfg, add_fc, masks=empty(masks_pre))
    g_pre, flips, total = _pinned(step.bufs_pre.pool, add_fc, lambda t: t[:ns * T].cpu(), lambda t: t[:ns].cpu(),
                                  masks_pre, plain, attn_frame != "none", False, ns * T)
    g_pre = afo.split_gates(g_pre, ns, T)[0]
    results, p1_64 = [], None
    for dtype in (torch.float64, torch.float32):
        q = {k: v.to(dtype) if v.dtype.is_floating_point else v for k, v in params.items()}
        x, y = xs.to(dtype), xt.to(dtype)
        update = _updater(kind)
        l1, g1 = pto.pretrain_step(q, x, labels, BETA, cfg, add_fc, train=drop > 0, masks=masks_pre, gates=g_pre)
        P = sorted(k for k, g in g1.items() if g is not None)
        pto.apply_update(q, g1, update, CLIP)
        if dtype == torch.float64:
            # the adaptation pass: its pattern on the weights the fp64 pre-training update left
            plain2 = afo.activation_pattern(q, x64, t64, BETA, cfg, add_fc, masks=masks)
            gates, f, n = _pinned(step.bufs.pool, add_fc, frames, videos, masks, plain2, True, True, (ns + nt) * T)
            flips, total = flips + f, total + n
            gates2 = None
            if ens == "MCD":
                k2 = None if masks2 is None else {"i_source": torch.ones(0, cfg.shared_dim, dtype=torch.uint8),
                                                  "v_source": torch.ones(0, cfg.video_dim, dtype=torch.uint8), **masks2}
                plain3 = orc.activation_pattern(q, x64[:0], t64, BETA, cfg, masks=k2)
                g3, f, n = _pinned(step.bufs2.pool, 1, lambda t: t[:nt * T].cpu(), lambda t: t[:nt].cpu(), masks2,
                                   plain3, attn_frame != "none", False, nt * T)
                _, gates2 = orc.split_gates(g3, 0, T)
                flips, total = flips + f, total + n
        l2, g2 = _adaptation(case, cfg, q, x, y, labels, masks, masks2, gates, gates2)
        pto.apply_update(q, g2, update, CLIP)
        results.append((l1, l2, P, g2, q))
    return results[0], results[1], flips, total


@gpu
@pytest.mark.parametrize("case", list(CASES))
def test_iteration_matches_fp64_oracle(case, engine):
    """One iteration against the fp64 oracle on the ReLU patterns the step realised in its passes: the pre-training
    loss, the set P it updates, the adaptation loss, its meter and its gradients (on the weights the pre-training
    update left), and each parameter's total change over both updates."""
    from tests.test_gpu_parity import FLIP_BOUND, NOISE_SCALE, PINNED_TOL, TOL
    from ta3n_b200.train import Adam, SGDNesterov, TrainStep, bucket_layout, stack_slots
    attn, attn_frame, ens, mu, add_fc, drop, (Bs, Bt), (ns, nt), extra, kind = CASES[case]
    if kind == "adam" and engine != "fp32":
        # Adam's normalised step turns the engine's rounding of near-zero gradient elements into parameter changes of
        # full size, so the adaptation pass runs on weights measurably off the oracle's; the Adam iteration is held to
        # fp32 here and to the stock torch.optim loop below
        pytest.skip("the chained Adam iteration is compared with the fp64 oracle on the fp32 engine")
    T = CASE_T.get(case, 5)
    m = _model(T=T, drop=drop, attn=attn, attn_frame=attn_frame, ens=ens, add_fc=add_fc)
    cfg = orc.PathConfig(num_class=7, num_segments=T, fc_dim=256, dropout_i=drop, dropout_v=drop, use_attn=attn,
                         use_attn_frame=attn_frame, ens_DA=ens)
    params = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    xs, xt, labels = _inputs(ns, nt, T)
    opt = SGDNesterov(lr=LR, clip_gradient=CLIP) if kind == "sgd" else Adam(lr=LR * 0.1, clip_gradient=CLIP)
    kw = {}
    if extra == "DAN":
        kw = dict(dis_DA="DAN", alpha=ALPHA)
    elif extra == "target_entropy":
        kw = dict(add_loss_DA="target_entropy")
    step = TrainStep(m, Bs, Bt, BETA, gamma=GAMMA, use_graph=False, mu=mu, optimizer=opt, pretrain_source=True,
                     stats=True, **kw)
    loss = step(xs.pin_memory(), xt.pin_memory(), labels).clone()
    torch.cuda.synchronize()
    key = int(step.step_counter.item())
    (l64, L64, P, g64, p64), (l32, L32, _, g32, p32), flips, total = \
        _oracle_iteration(case, cfg, params, xs, xt, labels, key, step, engine)
    assert flips <= max(FLIP_BOUND[engine] * total, 2), (flips, total)
    # P: the slots the pre-training update's mask covers are exactly the parameters its loss reaches
    names = {id(p): n for n, p in m.named_parameters()}
    _, offs, _, _ = bucket_layout(step.params, stack_slots(m))
    masked = sorted(names[id(p)] for j, p in enumerate(step.params) if step.pretrain_mask[offs[j]] != 0)
    assert masked == P, (masked, P)
    assert "fc_classifier_video_source.weight" in P and not any(n.startswith("fc_classifier_domain_video") for n in P)
    assert_close(step.loss_pre.cpu()[0], l64, TOL[engine], "pre-training loss", noise=abs(l32.double() - l64).item())
    assert_close(loss.cpu()[0], L64, TOL[engine], "adaptation loss", noise=abs(L32.double() - L64).item())
    st = step.stats()
    assert st.loss.count == 1 and st.loss.val == loss.item()         # the meter holds the adaptation pass's loss
    named = dict(m.named_parameters())
    for name, g in g64.items():
        if g is None:
            continue
        noise = (g32[name].double() - g).norm().item() * NOISE_SCALE[engine]
        assert_close(named[name].grad, g, PINNED_TOL[engine], f"grad {name}", noise=max(noise, 4e-9))
    # each parameter's change over both updates: normwise over the whole model, and per tensor where the change is
    # not negligible next to the largest (after the clip a small tensor's change carries the rounding of the large
    # gradients that set the coefficient)
    d_gpu, d64, d32 = {}, {}, {}
    for name, p0 in params.items():
        if name in named:
            d_gpu[name] = named[name].detach().cpu().double() - p0.double()
            d64[name], d32[name] = p64[name] - p0.double(), (p32[name] - p0).double()
    cat = lambda d: torch.cat([t.reshape(-1) for t in d.values()])      # noqa: E731
    noise = (cat(d32) - cat(d64)).norm().item() * NOISE_SCALE[engine]
    assert_close(cat(d_gpu), cat(d64), PINNED_TOL[engine], "update", noise=noise)
    biggest = max(t.norm().item() for t in d64.values())
    for name, d in d64.items():
        if d.norm().item() >= 1e-2 * biggest:
            noise = (d32[name] - d).norm().item() * NOISE_SCALE[engine]
            assert_close(d_gpu[name], d, PINNED_TOL[engine], f"update {name}", noise=max(noise, 1e-9))


def _stock_loss(outs, labels, ens, gamma, attn):
    from ta3n_b200 import loss as LS
    return LS.ta3n_loss(outs, labels, gamma, use_attn=attn)


@gpu
@pytest.mark.parametrize("attn,kind", [("TransAttn", "sgd"), ("none", "adam"), ("TransAttn", "adam")])
def test_three_iterations_match_the_stock_autograd_loop(attn, kind):
    """Three iterations against main.py:388-583 on this repo's VideoModel: autograd, clip_grad_norm_ and torch.optim
    SGD(nesterov=True) / Adam, with zero_grad() before each of the two updates.  The exported optimizer state equals
    the stock optimizer's (Adam: step 2k for P, k for the rest), and each loads into the other."""
    import ta3n_b200
    from ta3n_b200.train import Adam, SGDNesterov, TrainStep
    ta3n_b200.set_gemm_engine("fp32")
    try:
        xs, xt, labels = _inputs(8, 6, 5)
        m_a = _model(attn=attn)
        m_b = copy.deepcopy(m_a)
        cfg = SGDNesterov(lr=0.01, clip_gradient=0.5) if kind == "sgd" else Adam(lr=1e-3, clip_gradient=0.5)
        step = TrainStep(m_a, 8, 6, BETA, gamma=0.3, optimizer=cfg, pretrain_source=True)
        for _ in range(3):
            step(xs, xt, labels)
        torch.cuda.synchronize()
        params = list(m_b.parameters())
        if kind == "sgd":
            opt = torch.optim.SGD(params, 0.01, momentum=0.9, weight_decay=1e-4, nesterov=True)
        else:
            opt = torch.optim.Adam(params, 1e-3, weight_decay=1e-4)
        d = _dev()
        for _ in range(3):
            for pretrain in (True, False):
                opt.zero_grad(set_to_none=True)
                outs = m_b(xs.to(d), xt.to(d), list(BETA), 0, is_train=True, reverse=False)
                if pretrain:
                    loss = torch.nn.functional.cross_entropy(outs[1], labels.to(d))
                else:
                    loss = _stock_loss(outs, labels.to(d), "none", 0.3, attn)
                loss.backward()
                if pretrain:
                    # this repo's path is one autograd node: it returns zeros where the reference leaves .grad None
                    for p in params:
                        if p.grad is not None and not p.grad.any():
                            p.grad = None
                torch.nn.utils.clip_grad_norm_([p for p in params if p.grad is not None], 0.5)
                opt.step()
        pb = dict(m_b.named_parameters())
        for name, p in m_a.named_parameters():
            assert_close(p.detach(), pb[name].detach(), 1e-5, name)
        mine, theirs = step.optimizer_state_dict(), opt.state_dict()
        assert sorted(mine["state"]) == sorted(theirs["state"])
        for i, entry in theirs["state"].items():
            for k, v in entry.items():
                if k == "step":
                    assert float(mine["state"][i][k]) == float(v), (i, float(mine["state"][i][k]), float(v))
                else:
                    assert_close(mine["state"][i][k], v.cpu(), 1e-4, f"state[{i}][{k}]", noise=1e-9)
        if kind == "adam":
            assert {float(e["step"]) for e in theirs["state"].values()} == ({3.0, 6.0})
        stock = torch.optim.Adam(params, 1e-3, weight_decay=1e-4) if kind == "adam" else \
            torch.optim.SGD(params, 0.01, momentum=0.9, weight_decay=1e-4, nesterov=True)
        stock.load_state_dict(mine)
        step.load_optimizer_state_dict(theirs)
        again = step.optimizer_state_dict()
        assert {i: float(e["step"]) for i, e in again["state"].items() if "step" in e} == \
            {i: float(e["step"]) for i, e in theirs["state"].items() if "step" in e}
    finally:
        ta3n_b200.set_gemm_engine("tf32x3")


@gpu
@pytest.mark.parametrize("ens,kind", [("none", "adam"), ("MCD", "sgd")])
def test_eager_graph_reruns_and_resume_are_bit_identical(ens, kind):
    """Eager == graph == a second graph run over three iterations (dropout on, a short batch among them); and a run
    resumed from state_dict() after two of four iterations equals the uninterrupted run."""
    from ta3n_b200.train import Adam, SGDNesterov, TrainStep
    xs, xt, labels = _inputs(8, 6, 5)
    mk = lambda: SGDNesterov(lr=0.01) if kind == "sgd" else Adam(lr=1e-3)           # noqa: E731
    kw = dict(seed=11, gamma=0.3, mu=0.7 if ens == "MCD" else 0.0, pretrain_source=True)
    runs = []
    for use_graph in (False, True, True):
        m = _model(drop=0.5, ens=ens)
        step = TrainStep(m, 8, 6, BETA, use_graph=use_graph, optimizer=mk(), **kw)
        if use_graph:
            step.step_counter.fill_(0)       # the capture's warm-up advanced the dropout counter
        losses = []
        for i in range(3):
            n = (8, 6) if i != 1 else (5, 3)
            losses.append(step(xs[:n[0]], xt[:n[1]], labels[:n[0]]).clone())
            losses.append(step.loss_pre.clone())
        torch.cuda.synchronize()
        runs.append((torch.cat(losses), step.flat_param.clone()))
    for other in runs[1:]:
        assert torch.equal(runs[0][0], other[0]) and torch.equal(runs[0][1], other[1])

    m_a = _model(drop=0.5, ens=ens)
    m_b = copy.deepcopy(m_a)
    a = TrainStep(m_a, 8, 6, BETA, optimizer=mk(), **kw)
    for _ in range(4):
        a(xs, xt, labels)
    b0 = TrainStep(m_b, 8, 6, BETA, optimizer=mk(), **kw)
    for _ in range(2):
        b0(xs, xt, labels)
    sd = copy.deepcopy(b0.state_dict())
    params = copy.deepcopy(m_b.state_dict())
    m_c = _model(drop=0.5, ens=ens, seed=99)
    m_c.load_state_dict(params)
    c = TrainStep(m_c, 8, 6, BETA, optimizer=mk(), **kw)
    c.load_state_dict(sd)
    for _ in range(2):
        c(xs, xt, labels)
    torch.cuda.synchronize()
    assert torch.equal(a.flat_param, c.flat_param)


@gpu
def test_meters_are_the_adaptation_pass():
    """stats(): the loss meter takes the loss run() returns (the adaptation pass's) and top-1 the adaptation pass's
    logits of the real source rows, as main.py's AverageMeters do (main.py:418-583 updates them after the
    pre-training update)."""
    from oracle.train_stats_oracle import AverageMeter
    from ta3n_b200.train import SGDNesterov, TrainStep
    Bs = 8
    xs, xt, labels = _inputs(Bs, 6, 5)
    step = TrainStep(_model(drop=0.5), Bs, 6, BETA, optimizer=SGDNesterov(lr=0.01), stats=True, pretrain_source=True)
    ref_l, ref_1 = AverageMeter(), AverageMeter()
    for ns, nt in ((8, 6), (8, 6), (5, 2)):
        loss = step(xs[:ns], xt[:nt], labels[:ns]).item()
        logits = step.outputs[5][:ns].cpu()
        ref_l.update(loss)
        ref_1.update(100.0 * (logits.argmax(1) == labels[:ns]).sum().item() / ns, ns)
        assert step.loss_pre.item() != loss
    st = step.stats()
    assert st.loss.count == 3 and st.loss.avg == pytest.approx(ref_l.avg, rel=1e-6)
    assert st.top1.count == ref_1.count == 21 and st.top1.avg == pytest.approx(ref_1.avg, rel=1e-6)


@gpu
@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_launches_the_option_adds(kind):
    """The default step issues the launches it did before the option existed; the option adds the pre-training
    pass's own launches and one optimizer update (two under Adam: the adaptation update splits by step count)."""
    import ta3n_b200
    from ta3n_b200 import _lib
    from ta3n_b200 import functional as TF
    from tests.test_discrepancy import PLAIN_LAUNCHES
    from ta3n_b200.train import Adam, SGDNesterov, TrainStep
    ta3n_b200.set_gemm_engine("tf32x3")
    mk = lambda: SGDNesterov(lr=0.01) if kind == "sgd" else Adam(lr=1e-3)           # noqa: E731
    plain = TrainStep(_model(), 8, 6, BETA, optimizer=mk())
    step = TrainStep(_model(), 8, 6, BETA, optimizer=mk(), pretrain_source=True)
    if kind == "sgd":
        assert plain.launches_per_step == PLAIN_LAUNCHES[True]
    n0 = _lib.launch_count()
    scratch = step.bufs.workspace("forward_scratch", 48 << 20)
    _lib.load().ta3n_set_forward_scratch(TF._p(scratch), scratch.numel())
    try:
        step._enqueue_pretrain(_lib.load(), TF._stream(), False)
    finally:
        _lib.load().ta3n_set_forward_scratch(None, 0)
    torch.cuda.synchronize()
    pass_launches = _lib.launch_count() - n0
    opt_launches = 2 * (1 if kind == "sgd" else 2)
    assert step.launches_per_step == plain.launches_per_step + pass_launches + opt_launches, \
        (step.launches_per_step, plain.launches_per_step, pass_launches)
    # the eager step counts what it issued
    eager = TrainStep(_model(), 8, 6, BETA, optimizer=mk(), pretrain_source=True, use_graph=False)
    xs, xt, labels = _inputs(8, 6, 5)
    eager(xs, xt, labels)
    assert eager.launches_per_step == step.launches_per_step


@gpu
def test_device_sampler_is_bit_identical_to_load(tmp_path):
    """One gather feeds both updates: the sampler-fed step equals the load()-fed one, bit for bit, over two epochs
    with short last batches."""
    from ta3n_b200 import dataset as D
    from ta3n_b200.train import SGDNesterov, TrainStep
    from tests.test_device_sampler import _banks
    T, batch = 5, (8, 6)
    sets, banks = _banks(tmp_path, T, orc.FEATURE_DIM, (21, None), (9, 14), batch)
    model_a = _model(drop=0.5)
    model_b = copy.deepcopy(model_a)
    kw = dict(beta=BETA, gamma=0.3, seed=123, pretrain_source=True)
    sampler = D.DevicePairedSampler(banks[0], banks[1], batch, seed=4)
    step_a = TrainStep(model_a, *batch, sampler=sampler, optimizer=SGDNesterov(lr=0.01), **kw)
    step_b = TrainStep(model_b, *batch, optimizer=SGDNesterov(lr=0.01), **kw)
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
            assert torch.equal(loss_a, loss_b) and torch.equal(step_a.loss_pre, step_b.loss_pre), (epoch, n_step)
            assert torch.equal(step_a.flat_param, step_b.flat_param), (epoch, n_step)
            assert torch.equal(step_a.momentum_buf, step_b.momentum_buf), (epoch, n_step)
    assert n_step == 6


@gpu
def test_double_buffer_and_set_lr():
    """double_buffer=True with prefetch / swap equals the single-slot step, and set_lr sets the rate of both
    updates (lr 0: nothing moves)."""
    from ta3n_b200.train import SGDNesterov, TrainStep
    xs, xt, labels = _inputs(8, 6, 5)
    m_a = _model(drop=0.5)
    m_b = copy.deepcopy(m_a)
    kw = dict(seed=7, pretrain_source=True)
    a = TrainStep(m_a, 8, 6, BETA, optimizer=SGDNesterov(lr=0.01), **kw)
    b = TrainStep(m_b, 8, 6, BETA, optimizer=SGDNesterov(lr=0.01), double_buffer=True, **kw)
    a.step_counter.fill_(0)
    b.step_counter.fill_(0)
    b.load(xs, xt, labels)
    for i in range(3):
        a(xs, xt, labels)
        b.run()
        if i < 2:
            b.prefetch(xs, xt, labels)
            b.swap()
    torch.cuda.synchronize()
    assert torch.equal(a.flat_param, b.flat_param)
    a.set_lr(0.0)
    before = a.flat_param.clone()
    a(xs, xt, labels)
    torch.cuda.synchronize()
    assert torch.equal(before, a.flat_param)
