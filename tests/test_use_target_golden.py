"""use_target 'Sv' / 'none' against the unmodified reference.

CPU: the fp64 oracle (oracle/use_target_oracle.py) and ``loss.ta3n_loss(use_target=...)`` against the reference's
iterations (tests/golden/use_target_golden.npz, from oracle/gen_golden_use_target.py): losses, the parameters with a
gradient, the parameters after every update, the optimizer state with Adam's step counts, and the epoch meters; and
the oracle against the live reference where the tree is present.
GPU: one TrainStep iteration per golden case (its weights, inputs and options; dropout masks from the step's counter)
against the fp64 oracle on the ReLU patterns the step realised, on the fp32, tf32x3 and tf32 engines, with the
tolerances and noise rule of test_pretrain_source.py.
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle import add_fc_oracle as afo
from oracle import gen_golden_pretrain as gp
from oracle import gen_golden_use_target as G
from oracle import pretrain_oracle as pto
from oracle import ref_shims
from oracle import ta3n_oracle as orc
from oracle import use_target_oracle as uto
from tests.golden_util import assert_close
from tests.test_pretrain_source import _check_stored, _pinned, _real_masks, _unpack

gpu = pytest.mark.gpu


def _golden():
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "use_target_golden.npz"))
    return z, json.loads(bytes(z["meta_json"]).decode())


def _oracle_run(c, dtype=torch.float64):
    """The oracle's records of a golden case in the generator's format, plus ``loss.ta3n_loss`` on the oracle's
    outputs and each iteration's meters."""
    from ta3n_b200 import loss as LS
    from tests.optim_oracle import adam_step
    cfg = gp.case_config(c)
    p = {k: v.to(dtype) for k, v in gp.case_params(c).items()}
    xs, xt, labels = gp.case_inputs(c)
    ns, nt = c["ns"], c["nt"]
    xs, xt, labels = xs[:ns].to(dtype), xt[:nt].to(dtype), labels[:ns]
    lt = G.case_target_labels(c)[:nt]
    state, bufs = {}, {}
    if c["opt"] == "adam":
        update = lambda q, g: adam_step(q, g, state, gp.LR_ADAM)                          # noqa: E731
    else:
        update = lambda q, g: orc.sgd_nesterov_step(q, g, bufs, gp.LR_SGD, 0.9, 1e-4)     # noqa: E731
    runs = []
    for it in range(gp.ITERATIONS):
        rec = {}
        if c["pretrain"]:
            m_pre = _real_masks(c, gp.case_masks(c, it, 0), {"source": ns})
            loss, g = pto.pretrain_step(p, xs, labels, gp.BETA, cfg, c["add_fc"], masks=m_pre)
            pto.apply_update(p, g, update, gp.CLIP)
            rec["loss_pre"], rec["params_pre"] = loss.item(), {k: v.clone() for k, v in p.items()}
        m = _real_masks(c, gp.case_masks(c, it, 1), {"source": ns, "target": nt})
        with torch.no_grad():
            outs = afo.forward(p, xs, xt, gp.BETA, 0.0, cfg, c["add_fc"], masks=m)
        extra = c["extra"] if c["use_target"] == "Sv" else None
        if c["use_target"] == "Sv":
            loss, _, g = uto.sv_train_step(p, xs, xt, labels, lt, gp.BETA, cfg, c["add_fc"], gp.GAMMA, extra,
                                           gp.ALPHA, masks=m)
        else:
            loss, g = pto.pretrain_step(p, xs, labels, gp.BETA, cfg, c["add_fc"],
                                        masks={k: v for k, v in m.items() if k.endswith("_source")})
        rec["with_grad"] = sorted(k for k, v in g.items() if v is not None)
        rec["loss"] = loss.item()
        if extra != "DAN":
            add = "target_entropy" if extra == "target_entropy" else "attentive_entropy"
            rec["ta3n_loss"] = LS.ta3n_loss(outs, labels, gp.GAMMA, use_attn=c["use_attn"], add_loss_DA=add,
                                            use_target=c["use_target"], label_target=lt).item()
        rec["meters"] = uto.step_meters(outs, labels, lt, ns, nt, c["use_target"],
                                        attentive_entropy=c["use_attn"] != "none", gamma=gp.GAMMA)
        pto.apply_update(p, g, update, gp.CLIP)
        rec["params"] = {k: v.clone() for k, v in p.items()}
        if c["opt"] == "adam":
            rec["state"] = {k: {"step": float(st["step"]), "exp_avg": st["exp_avg"].clone(),
                                "exp_avg_sq": st["exp_avg_sq"].clone()} for k, st in state.items()}
        else:
            rec["state"] = {k: {"momentum_buffer": b.clone()} for k, b in bufs.items()}
        runs.append(rec)
    return runs


@pytest.mark.parametrize("name", list(G.CASES))
def test_oracle_equals_golden(name):
    """The oracle's iterations, ``loss.ta3n_loss`` and the oracle's epoch meters against the reference's."""
    z, meta = _golden()
    c = G.case(name)
    init = gp.case_params(c)
    runs = _oracle_run(c)
    for it, rec in enumerate(runs):
        k = f"{name}/{it}/"
        noise = meta[k + "noise"]
        assert rec["with_grad"] == sorted(meta[k + "with_grad"])
        keys = ("loss_pre", "loss") if c["pretrain"] else ("loss",)
        for key in keys:
            assert_close(torch.tensor(rec[key]), torch.tensor(meta[k + key]), 1e-5, k + key, noise=noise[key])
        if "ta3n_loss" in rec:
            assert_close(torch.tensor(rec["ta3n_loss"]), torch.tensor(meta[k + "loss"]), 1e-5, k + "ta3n_loss",
                         noise=noise["loss"])
        for part in (("params_pre", "params") if c["pretrain"] else ("params",)):
            stored = _unpack(z[k + part], meta[k + part + "/layout"])
            for n, t in stored.items():
                _check_stored(rec[part][n], t, init[n], 2e-4, f"{k}{part}/{n}", max(noise[part + "/" + n], 1e-9))
        stored = _unpack(z[k + "state"], meta[k + "state/layout"])
        assert sorted(rec["state"]) == sorted(meta[k + "state_names"])
        if c["opt"] == "adam":
            per_it = 2 if (c["pretrain"] or c["use_target"] == "none") else 1
            want = {n: (per_it if (c["pretrain"] and n in rec["with_grad"]) else 1) * (it + 1) for n in rec["state"]}
            assert {n: st["step"] for n, st in rec["state"].items()} == meta[k + "steps"] == want
        for key, t in stored.items():
            n, sk = key.rsplit("/", 1)
            _check_stored(rec["state"][n][sk], t, None, 2e-4 if sk != "exp_avg_sq" else 5e-4, f"{k}state/{key}",
                          max(noise["state/" + key], 1e-9))
    # the epoch's meters: main.py's AverageMeters over the reference's per-iteration values
    mine = uto.fold([r["meters"] for r in runs])
    from oracle.train_stats_oracle import AverageMeter
    want = {key: AverageMeter() for key in ("loss_c", "top1", "top5")}
    for it in range(gp.ITERATIONS):
        lc, p1, p5, n = meta[f"{name}/{it}/meters"]
        for key, v in (("loss_c", lc), ("top1", p1), ("top5", p5)):
            want[key].update(v, n)
    assert mine["loss_c"].count == want["loss_c"].count
    assert mine["loss_c"].avg == pytest.approx(want["loss_c"].avg, rel=1e-5)
    for key in ("top1", "top5"):
        assert mine[key].count == want[key].count and mine[key].avg == pytest.approx(want[key].avg, abs=1e-9)


@pytest.mark.skipif(not ref_shims.available(), reason="needs the reference tree")
@pytest.mark.parametrize("name", ["sv_attn", "sv_dan", "sv_short", "none_attn", "none_pretrain", "none_adam"])
def test_oracle_equals_live_reference(name):
    c = G.case(name)
    ref, _ = G.run_reference(c, torch.float64)
    mine = _oracle_run(c)
    for it, (r, o) in enumerate(zip(ref, mine)):
        assert sorted(r["with_grad"]) == o["with_grad"]
        assert o["loss"] == pytest.approx(r["loss"], rel=1e-9)
        for n, t in r["params"].items():
            assert_close(o["params"][n], t, 1e-9, f"{it} params/{n}", noise=1e-12)
        for n, st in r["state"].items():
            for sk, v in st.items():
                if sk == "step":
                    assert o["state"][n][sk] == float(v)
                else:
                    assert_close(o["state"][n][sk], v, 1e-8, f"{it} state/{n}/{sk}", noise=1e-12)


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------
@pytest.fixture(params=["fp32", "tf32x3", "tf32"])
def engine(request):
    import ta3n_b200
    ta3n_b200.set_gemm_engine(request.param)
    yield request.param
    ta3n_b200.set_gemm_engine("tf32x3")


def _empty_target(m):
    return None if m is None else {**m, **{k.replace("_source", "_target"): v[:0] for k, v in m.items()}}


@gpu
@pytest.mark.parametrize("name", list(G.CASES))
def test_iteration_matches_fp64_oracle(name, engine):
    """One TrainStep iteration of the golden case (dropout 0.5 from the step's counter) against the fp64 oracle on
    the ReLU patterns the step realised: the loss, every gradient and each parameter's total change."""
    from tests.test_gpu_parity import FLIP_BOUND, NOISE_SCALE, PINNED_TOL, TOL
    from ta3n_b200.models import VideoModel
    from ta3n_b200.train import Adam, SGDNesterov, TrainStep
    c = G.case(name)
    if c["opt"] == "adam" and engine != "fp32":
        pytest.skip("Adam's normalised step turns an engine's rounding of near-zero gradients into full-size weight "
                    "changes; the Adam iteration is compared with the fp64 oracle on the fp32 engine")
    if c["use_target"] == "none" and c["pretrain"] and engine != "fp32":
        pytest.skip("the two source passes of one iteration share their buffers, so the first pass's ReLU pattern "
                    "cannot be pinned; compared on the fp32 engine")
    T, add_fc, (Bs, Bt), (ns, nt) = c["T"], c["add_fc"], (c["bs"], c["bt"]), (c["ns"], c["nt"])
    cfg = gp.case_config(c)
    params = gp.case_params(c)
    m = VideoModel(c["C"], "video", "trn-m", "RGB", train_segments=T, val_segments=T, fc_dim=c["F"],
                   dropout_i=gp.DROPOUT, dropout_v=gp.DROPOUT, partial_bn=False, use_attn=c["use_attn"],
                   use_attn_frame=c["attn_frame"], add_fc=add_fc, verbose=False)
    m.load_state_dict(params, strict=False)
    m = m.to(torch.device("cuda:0")).train()
    xs, xt, labels = gp.case_inputs(c)
    xs, xt, labels = xs[:ns], xt[:nt], labels[:ns]
    lt = G.case_target_labels(c)[:nt]
    lr = gp.LR_SGD if c["opt"] == "sgd" else gp.LR_ADAM
    opt = SGDNesterov(lr=lr, clip_gradient=gp.CLIP) if c["opt"] == "sgd" else Adam(lr=lr, clip_gradient=gp.CLIP)
    kw = {}
    if c["extra"] == "DAN":
        kw = dict(dis_DA="DAN", alpha=gp.ALPHA, place_dis=gp.PLACE_DIS)
    elif c["extra"] == "target_entropy":
        kw = dict(add_loss_DA="target_entropy")
    sv = c["use_target"] == "Sv"
    step = TrainStep(m, Bs, Bt, gp.BETA, gamma=gp.GAMMA, use_graph=False, optimizer=opt,
                     pretrain_source=c["pretrain"], use_target=c["use_target"], **kw)
    loss = step(xs.pin_memory(), xt.pin_memory(), labels, lt if sv else None).clone()
    torch.cuda.synchronize()
    key = int(step.step_counter.item())
    F_, H = cfg.shared_dim, cfg.video_dim
    masks_pre = pto.pretrain_masks(key, Bs, T, F_, H, gp.DROPOUT, gp.DROPOUT, add_fc, ns=ns)
    if sv:
        masks = afo.train_step_masks(key, Bs, Bt, T, F_, H, gp.DROPOUT, gp.DROPOUT, add_fc, ns=ns, nt=nt)
    else:
        masks = uto.none_masks(key, Bs, T, F_, H, gp.DROPOUT, gp.DROPOUT, add_fc, ns=ns)
    x64, t64 = xs.double(), xt.double()
    p64 = {k: v.double() if v.dtype.is_floating_point else v for k, v in params.items()}
    src_rows = (lambda t: t[:ns * T].cpu(), lambda t: t[:ns].cpu())
    frame_disc = c["attn_frame"] != "none"
    flips = total = 0
    g_pre = None
    if c["pretrain"] and sv:
        plain = afo.activation_pattern(p64, x64, x64[:0], gp.BETA, cfg, add_fc, masks=_empty_target(masks_pre))
        g_pre, f, n = _pinned(step.bufs_pre.pool, add_fc, *src_rows, masks_pre, plain, frame_disc, False, ns * T)
        g_pre = afo.split_gates(g_pre, ns, T)[0]
        flips, total = flips + f, total + n
    results = []
    for dtype in (torch.float64, torch.float32):
        q = {k: v.to(dtype) if v.dtype.is_floating_point else v for k, v in params.items()}
        x, y = xs.to(dtype), xt.to(dtype)
        if c["opt"] == "adam":
            from tests.optim_oracle import adam_step
            state = {}
            update = lambda pp, gg, state=state: adam_step(pp, gg, state, lr)         # noqa: E731
        else:
            bufs = {}
            update = lambda pp, gg, bufs=bufs: orc.sgd_nesterov_step(pp, gg, bufs, lr, 0.9, 1e-4)   # noqa: E731
        if c["pretrain"]:
            _, g1 = pto.pretrain_step(q, x, labels, gp.BETA, cfg, add_fc, masks=masks_pre, gates=g_pre)
            pto.apply_update(q, g1, update, gp.CLIP)
        if dtype == torch.float64:
            if sv:
                plain2 = afo.activation_pattern(q, x64, t64, gp.BETA, cfg, add_fc, masks=masks)
                rows_f = lambda t: torch.cat([t[:ns * T], t[Bs * T:Bs * T + nt * T]]).cpu()    # noqa: E731
                rows_v = lambda t: torch.cat([t[:ns], t[Bs:Bs + nt]]).cpu()                    # noqa: E731
                gates, f, n = _pinned(step.bufs.pool, add_fc, rows_f, rows_v, masks, plain2, True, True,
                                      (ns + nt) * T)
            else:
                plain2 = afo.activation_pattern(q, x64, x64[:0], gp.BETA, cfg, add_fc, masks=_empty_target(masks))
                gates, f, n = _pinned(step.bufs_pre.pool, add_fc, *src_rows, masks, plain2, frame_disc, False, ns * T)
                gates = afo.split_gates(gates, ns, T)[0]
            flips, total = flips + f, total + n
        if sv:
            l2, _, g2 = uto.sv_train_step(q, x, y, labels, lt, gp.BETA, cfg, add_fc, gp.GAMMA, c["extra"], gp.ALPHA,
                                          masks=masks, gates=gates)
        else:
            l2, g2 = pto.pretrain_step(q, x, labels, gp.BETA, cfg, add_fc, masks=masks, gates=gates)
        pto.apply_update(q, g2, update, gp.CLIP)
        results.append((l2, g2, q))
    (L64, g64, p64u), (L32, g32, p32u) = results
    assert flips <= max(FLIP_BOUND[engine] * total, 2), (flips, total)
    assert_close(loss.cpu()[0], L64, TOL[engine], "loss", noise=abs(L32.double() - L64).item())
    named = dict(m.named_parameters())
    for pname, g in g64.items():
        if g is None:
            continue
        noise = (g32[pname].double() - g).norm().item() * NOISE_SCALE[engine]
        assert_close(named[pname].grad, g, PINNED_TOL[engine], f"grad {pname}", noise=max(noise, 4e-9))
    # under 'none' the slots outside P hold zero and the parameters there do not move
    if not sv:
        for pname, g in g64.items():
            if g is None and pname in named:
                assert torch.equal(named[pname].detach().cpu(), params[pname]), pname
    d_gpu, d64, d32 = {}, {}, {}
    for pname, p0 in params.items():
        if pname in named:
            d_gpu[pname] = named[pname].detach().cpu().double() - p0.double()
            d64[pname], d32[pname] = p64u[pname] - p0.double(), (p32u[pname] - p0).double()
    cat = lambda d: torch.cat([t.reshape(-1) for t in d.values()])      # noqa: E731
    noise = (cat(d32) - cat(d64)).norm().item() * NOISE_SCALE[engine]
    assert_close(cat(d_gpu), cat(d64), PINNED_TOL[engine], "update", noise=noise)
    biggest = max(t.norm().item() for t in d64.values())
    for pname, d in d64.items():
        if d.norm().item() >= 1e-2 * biggest:
            noise = (d32[pname] - d).norm().item() * NOISE_SCALE[engine]
            assert_close(d_gpu[pname], d, PINNED_TOL[engine], f"update {pname}", noise=max(noise, 1e-9))
