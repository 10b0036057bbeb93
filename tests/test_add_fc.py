"""Stacked shared frame layers (add_fc 2 and 3, models.py:141-153, 565-603).

CPU: the product's parameters (names, shapes, initial values under a seed) equal the reference's, a reference
state_dict loads, the oracle (``oracle/add_fc_oracle.py``) equals the reference's stored results
(``tests/golden/add_fc_golden.npz``, ``oracle/gen_golden_add_fc.py``), and the options outside the path are refused.
GPU: ``ta3n_shared_fc_bwd_dx`` against fp64 at fp32 grade, and VideoModel / EvalStep against the fixture and the
oracle, on every GEMM engine.
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle import add_fc_oracle as afo
from oracle import gen_golden_add_fc as gen
from oracle import ta3n_oracle as orc
from tests.golden_util import STRUCTURAL_ZERO_GRADS, TOL_FP32, TOL_PATH, assert_close

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "add_fc_golden.npz")
Z = np.load(GOLDEN)
META = json.loads(bytes(Z["meta_json"]).decode())
CASES = list(gen.CASES)
ENGINES = ["fp32", "tf32x3", "tf32"]
NOISE_SCALE = {"fp32": 1.0, "tf32x3": 8.0}      # as tests/test_gpu_parity.py: 8 x NOISE_SCALE x the reference's noise


def product_model(c, device="cpu"):
    """The product VideoModel of a fixture case, built under the case's seed (its init is the reference's)."""
    from ta3n_b200.models import VideoModel
    torch.manual_seed(gen.MODEL_SEED)
    m = VideoModel(c["C"], "video", c.get("agg", "trn-m"), "RGB", train_segments=c["T"], val_segments=c["T"],
                   add_fc=c["add_fc"], fc_dim=c["F"], dropout_i=gen.DROPOUT, dropout_v=gen.DROPOUT, partial_bn=False,
                   use_attn=c["use_attn"], use_attn_frame=c["attn_frame"], verbose=False)
    return m.to(device)


def perturbed_params(c):
    sd = {k: v.detach().clone() for k, v in product_model(c).state_dict().items()}
    gen.perturb_(sd)
    return sd


def pinned(key):
    """(whole tensor or None, stats or None, sample or None) of a stored result."""
    if key in Z.files:
        return Z[key], None, None
    return None, Z[key + "#stats"], Z[key + "#sample"]


def assert_pinned(t, key, tol, what, noise=0.0):
    t = t.detach().double().cpu()
    whole, stats, samp = pinned(key)
    if whole is not None:
        assert tuple(t.shape) == whole.shape, (what, tuple(t.shape), whole.shape)
        return assert_close(t, whole, tol, what, noise)
    s, n = stats
    flat = t.reshape(-1)
    assert abs(flat.norm().item() - n) <= tol * n + 8 * noise, f"{what}: norm {flat.norm().item():.6e} vs {n:.6e}"
    return assert_close(flat[::META["stride"]], samp, tol * 4, what + " (sample)", noise)


def check_against_fixture(case, loss, outs, grads, tol, noise_scale=1.0):
    """loss, every output of the 10-tuple and every parameter gradient against the reference's stored values."""
    k = case + "/"
    assert abs(float(loss) - float(Z[k + "loss"])) <= tol * abs(float(Z[k + "loss"])) + 8 * float(Z[k + "noise/loss"])
    flat = gen.flat_outputs(outs)
    assert len(flat) == META["n_out"][case]
    for i, t in enumerate(flat):
        assert_pinned(t, k + f"out/{i}", tol, f"{case}: output {i}", float(Z[k + f"noise/out/{i}"]) * noise_scale)
    used = META["used_params"][case]
    assert sorted(used) == sorted(n for n, g in grads.items() if g is not None), case
    for name in used:
        if name in STRUCTURAL_ZERO_GRADS:
            assert grads[name].double().norm().item() <= 1e-6
            continue
        noise = max(float(Z[k + "noise/grad/" + name]), 4e-9) * noise_scale
        assert_pinned(grads[name], k + "grad/" + name, tol, f"{case}: grad {name}", noise)


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES)
def test_parameters_equal_the_reference_init(case):
    """State-dict keys in the reference's order, shapes and values under the seed: the stacked layers are created
    right after the first one, so every later tensor shifts the same way."""
    c = gen.CASES[case]
    sd = product_model(c).state_dict()
    want = META["state_keys"][case]
    assert [[k, list(v.shape)] for k, v in sd.items()] == want
    for key, v in sd.items():
        if not v.dtype.is_floating_point:
            continue
        whole, stats, samp = pinned(f"{case}/init/{key}")
        if whole is not None:
            assert torch.equal(v.float(), torch.from_numpy(whole)), key
        else:
            d = v.double().reshape(-1)
            assert abs(d.sum().item() - stats[0]) <= 1e-9 * max(1.0, stats[1]), key
            assert abs(d.norm().item() - stats[1]) <= 1e-9 * max(1.0, stats[1]), key
            assert torch.equal(v.float().reshape(-1)[::META["stride"]], torch.from_numpy(samp)), key


@pytest.mark.parametrize("case", ["transattn_fc3", "avgpool_fc3"])
def test_reference_state_dict_loads(case):
    c = gen.CASES[case]
    ref_sd = {k: torch.full(shape, 0.25) for k, shape in META["state_keys"][case]}
    m = product_model(c)
    m.load_state_dict(ref_sd, strict=True)
    assert torch.equal(m.fc_feature_shared_3_source.weight, ref_sd["fc_feature_shared_3_source.weight"])


@pytest.mark.parametrize("case", CASES)
def test_oracle_equals_reference(case):
    """The stacked oracle, in fp32, equals the unmodified reference: outputs, the longer feature lists, every gradient
    (with the injected per-layer masks in the training cases)."""
    c = gen.CASES[case]
    cfg, xs, xt, labels, masks = gen.case_inputs(c)
    params = perturbed_params(c)
    loss, outs, grads = afo.train_step(params, xs, xt, labels, gen.BETA, cfg, c["add_fc"], gen.GAMMA,
                                       train=c["train"], masks=masks, lower_weight=gen.LOWER_WEIGHT)
    assert len(outs[4]) == 2 + c["add_fc"] and len(outs[9]) == 2 + c["add_fc"]
    check_against_fixture(case, loss, outs, grads, TOL_FP32)


def test_oracle_gates_reproduce_the_relu_forward():
    """On the realised pattern (activation_pattern as gates) the oracle computes what it computes with ReLUs."""
    c = gen.CASES["transattn_fc3"]
    cfg, xs, xt, labels, masks = gen.case_inputs(c)
    params = {k: v.double() if v.dtype.is_floating_point else v for k, v in perturbed_params(c).items()}
    xs, xt = xs.double(), xt.double()
    gates = afo.activation_pattern(params, xs, xt, gen.BETA, cfg, 3, masks)
    assert {"shared", "shared2", "shared3"} <= set(gates)
    a = afo.forward(params, xs, xt, gen.BETA, 0.0, cfg, 3, masks=masks)
    b = afo.forward(params, xs, xt, gen.BETA, 0.0, cfg, 3, masks=masks, gates=gates)
    for x, y in zip(gen.flat_outputs(a), gen.flat_outputs(b)):
        assert torch.allclose(x, y, rtol=1e-12, atol=1e-15)


def test_options_outside_the_path_are_refused():
    from ta3n_b200.models import VideoModel
    with pytest.raises(NotImplementedError, match="add_fc"):
        VideoModel(5, "video", "trn-m", "RGB", add_fc=4, verbose=False)
    with pytest.raises(ValueError):
        VideoModel(5, "video", "trn-m", "RGB", add_fc=0, verbose=False)


def test_add_fc_1_parameters_are_unchanged():
    """At add_fc=1 the operator's parameter list is what it always was (no stacked tensors)."""
    from ta3n_b200.models import VideoModel
    for agg, n in (("trn-m", 6 + 6 * 4 + 6), ("avgpool", 12)):
        m = VideoModel(5, "video", agg, "RGB", add_fc=1, fc_dim=256, verbose=False)
        assert len(m.path_parameters()) == n
        m3 = VideoModel(5, "video", agg, "RGB", add_fc=3, fc_dim=256, verbose=False)
        p3 = m3.path_parameters()
        assert len(p3) == n + 4
        assert p3[n] is m3.fc_feature_shared_2_source.weight and p3[n + 3] is m3.fc_feature_shared_3_source.bias


# ---------------------------------------------------------------------------------------------------------------------
# GPU: the new entry point at fp32 grade
# ---------------------------------------------------------------------------------------------------------------------
def _bwd_dx_case(rows_s, rows_t, F, p, ext, exact, seed):
    from tests.test_tc_tf32_kernel import grid, tf32_exact
    g = torch.Generator().manual_seed(seed)
    rows = rows_s + rows_t
    if exact:
        x = grid((rows, F), 4, g, relu=True)             # the layer below's output: non-negative, many zeros
        W = grid((F, F), 5, g)
        feat = grid((rows, F), 4, g, relu=True)
        dfeat = grid((rows, F), 6, g)
        gext = grid((rows, F), 6, g) if ext else None
    else:
        x = torch.randn(rows, F, generator=g).clamp_min(0.0)
        W = torch.randn(F, F, generator=g)
        feat = torch.randn(rows, F, generator=g).clamp_min(0.0)
        dfeat = torch.randn(rows, F, generator=g)
        gext = torch.randn(rows, F, generator=g) if ext else None
    dpre = (dfeat.double() + (0 if gext is None else gext.double())) * (feat > 0) / (1.0 - p)
    if exact:
        assert bool((tf32_exact(dpre.float()).double() == dpre).all()) and bool((tf32_exact(W) == W).all())
    return x, W, feat, dfeat, gext, dpre


BWD_DX = [(1001, 1503, 512, 0.5, True), (0, 777, 1024, 0.0, False), (640, 640, 250, 0.5, True),
          (2560, 2560, 512, 0.0, True), (37, 0, 1024, 0.5, False), (0, 0, 512, 0.0, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("exact", [True, False], ids=["tierE", "tierR"])
@pytest.mark.parametrize("rows_s,rows_t,F,p,ext", BWD_DX, ids=[f"{c[0]}+{c[1]}-F{c[2]}-p{c[3]}-ext{int(c[4])}"
                                                               for c in BWD_DX])
def test_shared_fc_bwd_dx(rows_s, rows_t, F, p, ext, exact, engine):
    """dpre written into dfeat exactly; dx = dpre W, dW = dpre^T x, db = colsum(dpre) against fp64.  Tier E
    (tf32-exact operands): 2e-5 normwise and per 128 x 128 tile on every engine and route (F = 250 is not a 16-byte
    row stride: the SIMT fallback).  Tier R (raw randn operands) on the plain engine: round to nearest."""
    import ta3n_b200
    from ta3n_b200 import _lib as L
    from tests.test_tc_tf32_kernel import TIER_E, tier_e, tier_r
    from tests.test_x3_kernel import _Out
    if not exact and engine != "tf32":
        pytest.skip("tier R is the plain tensor-core engine's check")
    ta3n_b200.set_gemm_engine(engine)
    try:
        lib = L.load()
        d = torch.device("cuda:0")
        rows = rows_s + rows_t
        x, W, feat, dfeat, gext, dpre = _bwd_dx_case(rows_s, rows_t, F, p, ext, exact, rows + F + int(exact))
        x_d, W_d, feat_d, dfeat_d = x.to(d), W.to(d), feat.to(d), dfeat.to(d)
        gext_d = None if gext is None else gext.to(d)
        dfb = torch.empty_like(dfeat_d)
        dx, dW, db = _Out(max(rows, 1), F), _Out(F, F), _Out(F)
        ws = torch.empty(max(256, lib.ta3n_shared_fc_bwd_workspace_bytes(rows, F, F)), dtype=torch.uint8, device=d)

        def run():
            dfb.copy_(dfeat_d)
            for o in (dx, dW, db):
                o.t.fill_(float("nan"))
            L.check(lib.ta3n_shared_fc_bwd_dx(
                x_d.data_ptr(), rows_s, x_d[rows_s:].data_ptr(), rows_t, F, F, W_d.data_ptr(), feat_d.data_ptr(),
                dfb.data_ptr(), None if gext_d is None else gext_d.data_ptr(), p, dx.ptr(), dW.ptr(), db.ptr(),
                ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream))

        run()
        torch.cuda.synchronize()
        first = [t.t.clone() for t in (dx, dW, db)]
        run()
        torch.cuda.synchronize()
        for a, o in zip(first, (dx, dW, db)):
            assert torch.equal(a.nan_to_num(7.0), o.t.nan_to_num(7.0)), "a second run gave a different result"
        for o, w in ((dx, "dx"), (dW, "dW"), (db, "db")):
            o.check_guard(w)
        if rows == 0:
            assert torch.equal(dW.t, torch.zeros_like(dW.t)) and torch.equal(db.t, torch.zeros_like(db.t))
            assert dx.t.isnan().all(), "dx has no rows: nothing may be written"
            return
        assert torch.equal(dfb.double().cpu(), dpre.float().double()), "dpre (written into dfeat)"
        what = f"rows={rows_s}+{rows_t} F={F} p={p} {engine}"
        want_dx = dpre.to(d) @ W.to(d, torch.float64)
        want_dW = dpre.t().to(d) @ x.to(d, torch.float64)
        if exact:
            tier_e("dx " + what, dx.t, want_dx)
            tier_e("dW " + what, dW.t, want_dW)
        else:
            tier_r("dx " + what, dx.t, want_dx)
            tier_r("dW " + what, dW.t, want_dW)
        want_db = dpre.sum(0).to(d)
        err = ((db.t.double() - want_db).norm() / want_db.norm()).item()
        assert err <= TIER_E, f"db {what}: {err:.2e}"
    finally:
        ta3n_b200.set_gemm_engine("tf32x3")


@pytest.mark.gpu
def test_shared_fc_bwd_dx_defers_only_the_weight_gradient():
    """Between ta3n_wgrad_defer_begin and _flush, dx is complete before the flush; dW, db arrive with it."""
    from ta3n_b200 import _lib as L
    lib = L.load()
    d = torch.device("cuda:0")
    rows_s, rows_t, F = 640, 512, 512
    x, W, feat, dfeat, gext, dpre = _bwd_dx_case(rows_s, rows_t, F, 0.5, True, True, 3)
    x_d, W_d, feat_d, dfb = x.to(d), W.to(d), feat.to(d), dfeat.to(d)
    dx = torch.full((rows_s + rows_t, F), float("nan"), device=d)
    dW = torch.full((F, F), float("nan"), device=d)
    db = torch.full((F,), float("nan"), device=d)
    ws = torch.empty(lib.ta3n_shared_fc_bwd_workspace_bytes(rows_s + rows_t, F, F), dtype=torch.uint8, device=d)
    fws = torch.empty(lib.ta3n_wgrad_defer_workspace_bytes(), dtype=torch.uint8, device=d)
    st = torch.cuda.current_stream().cuda_stream
    L.check(lib.ta3n_wgrad_defer_begin())
    L.check(lib.ta3n_shared_fc_bwd_dx(x_d.data_ptr(), rows_s, x_d[rows_s:].data_ptr(), rows_t, F, F, W_d.data_ptr(),
                                      feat_d.data_ptr(), dfb.data_ptr(), gext.to(d).data_ptr(), 0.5, dx.data_ptr(),
                                      dW.data_ptr(), db.data_ptr(), ws.data_ptr(), ws.numel(), st))
    torch.cuda.synchronize()
    assert not dx.isnan().any() and dW.isnan().all() and db.isnan().all()
    L.check(lib.ta3n_wgrad_defer_flush(fws.data_ptr(), fws.numel(), st))
    torch.cuda.synchronize()
    want = dpre.t().to(d) @ x.to(d, torch.float64)
    assert ((dW.double() - want).norm() / want.norm()).item() <= 2e-5
    assert not db.isnan().any()


# ---------------------------------------------------------------------------------------------------------------------
# GPU: VideoModel and EvalStep
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(params=ENGINES)
def engine(request):
    import ta3n_b200
    ta3n_b200.set_gemm_engine(request.param)
    yield request.param
    ta3n_b200.set_gemm_engine("tf32x3")


def _cat_masks(masks, add_fc):
    out = {"v": torch.cat([masks["v_source"], masks["v_target"]], 0)}
    for layer in range(1, add_fc + 1):
        k = "i" if layer == 1 else f"i{layer}"
        out[k] = torch.cat([masks[k + "_source"], masks[k + "_target"]], 0)
    return out


def _run_model(c, params, cfg, xs, xt, labels, masks):
    from ta3n_b200.loss import ta3n_loss
    d = torch.device("cuda:0")
    model = product_model(c, d)
    model.load_state_dict(params)
    if c["train"]:
        model.train()
        model.dropout_masks = _cat_masks(masks, c["add_fc"])
    else:
        model.eval()
    outs = model(xs.to(d), xt.to(d), list(gen.BETA), 0, is_train=True, reverse=False)
    loss = ta3n_loss(outs, labels.to(d), gen.GAMMA, use_attn=c["use_attn"]) + afo.lower_feature_loss(outs,
                                                                                                     gen.LOWER_WEIGHT)
    loss.backward()
    grads = {n: (None if p.grad is None else p.grad.detach().cpu()) for n, p in model.named_parameters()}
    return model, loss.detach().cpu(), outs, grads


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_model_matches_reference_fixture(case, engine):
    """VideoModel with 2 and 3 shared layers against the reference's stored results within TOL_PATH (plus the
    reference's own rounding noise), including the gradient of a loss on the lower layers' outputs.  On the engines
    whose forward is fp32 grade: plain tf32 flips ReLU units of these (non-degenerate) weights, and a flip moves a
    gradient by O(1) -- that engine is held to the fp64 pattern's units in the test below."""
    if engine == "tf32":
        pytest.skip("plain tf32 is not fp32 grade in the forward")
    c = gen.CASES[case]
    cfg, xs, xt, labels, masks = gen.case_inputs(c)
    params = perturbed_params(c)
    _, loss, outs, grads = _run_model(c, params, cfg, xs, xt, labels, masks)
    outs = tuple(o if not isinstance(o, list) else [t.detach().cpu() for t in o] for o in outs)
    outs = tuple(o.detach().cpu() if torch.is_tensor(o) else o for o in outs)
    check_against_fixture(case, loss, outs, grads, TOL_PATH, noise_scale=NOISE_SCALE[engine])


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["transattn_fc3", "attnframe_t7_fc2", "noattn_fc2"])
def test_model_matches_fp64_oracle_on_realised_pattern(case, engine):
    """Gradients against the fp64 oracle evaluated on the ReLU pattern the product realised in every shared layer
    (the fp64 pattern elsewhere), on the fp32-grade engines: at most 5e-6 of the shared units may differ from the
    fp64 pattern."""
    if engine == "tf32":
        pytest.skip("plain tf32 also flips units behind the shared layers, which this pattern does not pin")
    c = gen.CASES[case]
    cfg, xs, xt, labels, masks = gen.case_inputs(c)
    params = perturbed_params(c)
    _, loss, outs, grads = _run_model(c, params, cfg, xs, xt, labels, masks)
    p64 = {k: v.double() if v.dtype.is_floating_point else v for k, v in params.items()}
    gates = afo.activation_pattern(p64, xs.double(), xt.double(), gen.BETA, cfg, c["add_fc"], masks)
    L = c["add_fc"]
    realised = {}
    flip, total = 0, 0
    for layer in range(1, L + 1):
        key = "shared" if layer == 1 else f"shared{layer}"
        ff = torch.cat([outs[4][2 + L - layer], outs[9][2 + L - layer]], 0).detach().reshape(-1, cfg.shared_dim).cpu()
        keep = _cat_masks(masks, L)["i" if layer == 1 else f"i{layer}"].bool() if masks else torch.ones_like(ff).bool()
        on = ff > 0
        # where dropout zeroed a unit its sign is not visible: take the fp64 pattern there
        got = torch.where(keep, on, gates[key])
        flip += int((got != gates[key]).sum())
        total += got.numel()
        realised[key] = got
    assert flip <= 5e-6 * total + 1, f"{flip} of {total} shared units changed state"
    gates.update(realised)
    loss64, outs64, grads64 = afo.train_step(p64, xs.double(), xt.double(), labels, gen.BETA, cfg, L, gen.GAMMA,
                                             train=c["train"], masks=masks, gates=gates,
                                             lower_weight=gen.LOWER_WEIGHT)
    tol = TOL_PATH
    for name, g64 in grads64.items():
        if g64 is None or name in STRUCTURAL_ZERO_GRADS:
            continue
        noise = max(float(Z[f"{case}/noise/grad/{name}"]), 4e-9) * NOISE_SCALE[engine]
        assert_close(grads[name], g64, tol, f"{case}: grad {name} vs fp64 oracle", noise)


@pytest.mark.gpu
@pytest.mark.parametrize("agg", ["trn-m", "avgpool"])
def test_eval_step_with_stacked_layers(tmp_path, agg, engine):
    """EvalStep at add_fc=2, through host batches and through the device sampler (a short last batch): the logits equal
    VideoModel.forward(val, val, is_train=False) and the two routes are bit-identical."""
    from ta3n_b200 import dataset as D
    from ta3n_b200.evaluate import EvalStep
    from ta3n_b200.models import VideoModel
    from tests.test_eval_step import _shard
    T, B, C = 5, 8, 6
    ds = _shard(tmp_path, "v", 21, T, 2048, 3, n_class=C)                 # 8 + 8 + 5
    torch.manual_seed(5)
    m = VideoModel(C, "video", agg, "RGB", train_segments=T, val_segments=T, add_fc=2, fc_dim=256,
                   partial_bn=False, verbose=False).cuda().eval()
    with torch.no_grad():
        for k, v in m.named_parameters():
            if "weight" in k:
                v.add_(0.02 * torch.randn_like(v))
    ev_dev = EvalStep(m, B, sampler=D.DeviceEvalSampler(D.DeviceFeatureBank(ds), B), keep_scores=True)
    ev_host = EvalStep(m, B, keep_scores=True, epoch_rows=len(ds))
    r_dev = ev_dev.run_epoch()
    data = torch.from_numpy(np.stack([ds[i][0].numpy() for i in range(len(ds))]))
    labels = torch.from_numpy(ds.labels[:len(ds)])
    for a in range(0, len(ds), B):
        ev_host(data[a:a + B], labels[a:a + B])
    r_host = ev_host.result()
    assert r_dev.n == r_host.n == 21 and r_dev.correct == r_host.correct
    assert torch.equal(r_dev.scores, r_host.scores)
    want = []
    with torch.no_grad():
        for a in range(0, len(ds), B):
            x = data[a:a + B].cuda()
            want.append(m(x, x, [0.0, 0.0, 0.0], 0, is_train=False, reverse=False)[1].cpu())
    want = torch.cat(want)
    # VideoModel.forward runs 2B rows (val, val), EvalStep B: the GEMM schedules differ, so equal to fp32 rounding on the
    # fp32-grade engines and to the path's budget under plain tf32
    err = ((r_host.scores.cpu().double() - want.double()).norm() / want.double().norm()).item()
    assert err <= (TOL_PATH if engine == "tf32" else 1e-5), f"EvalStep logits vs VideoModel.forward: {err:.2e}"
    # the eval oracle (validate()'s loss / top-k / confusion) on the fp64 stacked oracle's logits
    from oracle import eval_oracle as eo
    cfg = orc.PathConfig(num_class=C, num_segments=T, fc_dim=256, dropout_i=0.0, dropout_v=0.0,
                         frame_aggregation=agg)
    p64 = {k: v.detach().double().cpu() if v.dtype.is_floating_point else v.cpu() for k, v in m.state_dict().items()}
    z64 = afo.forward(p64, data.double(), data.double(), [0.0, 0.0, 0.0], 0.0, cfg, 2, train=False)[1]
    assert_close(r_host.scores.cpu(), z64, 1e-5 if engine != "tf32" else TOL_PATH, "EvalStep logits vs fp64 oracle")
    ref = eo.epoch_metrics(z64.numpy(), labels.numpy(), B, topk=(1, 5))
    assert r_host.n == ref["n"] and r_host.batches == 3
    assert r_host.loss == pytest.approx(ref["loss"], rel=1e-4 if engine != "tf32" else 2e-3)
    margins = eo.topk_margin(z64.numpy(), labels.numpy(), 1)
    n_close = int((margins < 1e-3 * np.abs(z64.numpy()).max()).sum())
    assert abs(r_host.correct[0] - ref["correct"][0]) <= n_close
