"""TrainStep with add_loss_DA='target_entropy': gamma * the mean entropy of the target predictions (main.py:541-545,
loss.py:8-12) as one CUDA loss launch in the captured step.

CPU: the oracle (oracle/target_entropy_oracle.py) against the reference's iteration (tests/golden/
target_entropy_golden.npz, and the live reference where it is present), the options TrainStep refuses, the C ABI's
argument checks.
GPU: the entry alone against fp64 at fp32 grade (rows past the warps' first pass, classes past the lanes' first trip,
clamped / absent valid_rows, underflowing and uniform rows, accumulation over launches); one step against the fp64
oracle on every engine (dropout off and on, MCD with mu 0 and 0.7, with DAN, short batches), a batch
with no target row against the step without the term, three SGD steps against the stock autograd loop, bit-identical
reruns / eager vs graph / resume, the meters, and the launches the term adds.
"""
import copy
import json
import os

import numpy as np
import pytest
import torch

from oracle import gen_golden_target_entropy as gen
from oracle import mcd_oracle as mcd
from oracle import ref_shims
from oracle import ta3n_oracle as orc
from oracle import target_entropy_oracle as teo
from tests.golden_util import TOL_FP32, assert_close

gpu = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
BETA = (0.75, 0.6, 0.5)


def _golden():
    z = np.load(os.path.join(HERE, "golden", "target_entropy_golden.npz"))
    return z, json.loads(bytes(z["meta_json"]).decode())


def _stored(t, z, key, tol, what, noise=0.0):
    t = t.detach().double().cpu()
    if key in z.files:
        assert tuple(t.shape) == z[key].shape, (what, tuple(t.shape), z[key].shape)
        assert_close(t, z[key], tol, what, noise=noise)
        return
    s, n = z[key + "#stats"]
    flat = t.reshape(-1)
    assert abs(flat.norm().item() - n) <= tol * n + 8 * noise, f"{what}: norm {flat.norm().item():.6e} vs {n:.6e}"
    assert_close(flat[::gen.gm.STRIDE], z[key + "#sample"], tol * 4, what + " (sample)", noise=noise)


def _case(name, order):
    c = gen.CASES[name]
    cfg, xs, xt, labels, m1, m2 = gen.case_inputs(c)
    params = orc.init_params(cfg, seed=gen.gm.MODEL_SEED)
    gen.gm.perturb(params, order)
    return c, cfg, params, xs, xt, labels, m1, m2


def _oracle(c, cfg, params, xs, xt, labels, m1, m2):
    return teo.entropy_train_step(params, xs, xt, labels, gen.BETA, cfg, gen.GAMMA, masks=m1, mu=c["mu"],
                                  masks2={"i_target": m2["i_target"], "v_target": m2["v_target"]})


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(gen.CASES))
def test_oracle_equals_golden(case):
    """Loss, the unscaled term and every gradient of the reference's iteration with --add_loss_DA target_entropy
    (TransAttn / none / frame attention, and MCD, whose term reads pass 1's target logits)."""
    z, meta = _golden()
    k = case + "/"
    c, cfg, params, xs, xt, labels, m1, m2 = _case(case, meta[k + "param_order"])
    loss, term, grads = _oracle(c, cfg, params, xs, xt, labels, m1, m2)
    assert_close(loss, z[k + "loss"], TOL_FP32, f"{case} loss", noise=float(z[k + "noise/loss"]))
    assert_close(term, z[k + "term"], TOL_FP32, f"{case} term", noise=float(z[k + "noise/term"]))
    with_grad = meta[k + "with_grad"]
    assert sorted(n for n, g in grads.items() if g is not None) == sorted(with_grad)
    for n in with_grad:
        _stored(grads[n], z, k + "grad/" + n, 2e-4, f"{case} grad {n}",
                noise=max(float(z[k + "grad_noise/" + n]), 4e-9))


@pytest.mark.skipif(not ref_shims.available(), reason="needs the reference tree")
@pytest.mark.parametrize("case", ["attn", "mcd_mu07"])
def test_oracle_equals_live_reference(case):
    model, order, loss, term = gen.run_reference(gen.CASES[case])
    c, cfg, params, xs, xt, labels, m1, m2 = _case(case, order)
    got, got_term, grads = _oracle(c, cfg, params, xs, xt, labels, m1, m2)
    assert_close(got, loss.detach(), TOL_FP32, "loss")
    assert_close(got_term, term.detach(), TOL_FP32, "term")
    for n, p in model.named_parameters():
        if p.grad is not None:
            assert_close(grads[n], p.grad, 2e-4, f"grad {n}", noise=1e-8)


def test_torch_loss_adds_the_term():
    """ta3n_b200.loss.ta3n_loss (the autograd path) adds gamma * the term, and nothing for an empty target half."""
    from ta3n_b200.loss import ta3n_loss
    g = torch.Generator().manual_seed(0)
    out_s, out_t, lab = torch.randn(4, 6, generator=g), torch.randn(3, 6, generator=g), torch.arange(4) % 6
    pd = [torch.randn(4, 2, generator=g) for _ in range(3)], [torch.randn(3, 2, generator=g) for _ in range(3)]
    outs = (None, out_s, None, pd[0], None, None, out_t, None, pd[1], None)
    base = ta3n_loss(outs, lab, 0.5, add_loss_DA="none")
    assert ta3n_loss(outs, lab, 0.5, add_loss_DA="target_entropy").item() == \
        pytest.approx(base.item() + 0.5 * teo.target_entropy(out_t).item(), rel=1e-6)
    empty = (None, out_s, None, pd[0], None, None, out_t[:0], None, [p[:0] for p in pd[1]], None)
    assert ta3n_loss(empty, lab, 0.5, add_loss_DA="target_entropy").item() == \
        ta3n_loss(empty, lab, 0.5, add_loss_DA="none").item()


def _cpu_model(**kw):
    from ta3n_b200.models import VideoModel
    args = dict(train_segments=5, val_segments=5, fc_dim=64, verbose=False)
    args.update(kw)
    return VideoModel(5, "video", "trn-m", "RGB", **args).train()


@pytest.mark.parametrize("ens", ["none", "MCD"])
def test_train_step_refusals(ens):
    from ta3n_b200 import Ta3nError
    from ta3n_b200.train import TrainStep
    m = _cpu_model(ens_DA=ens)
    for bad in ("attentive", "target", "entropy", "", None):
        with pytest.raises(ValueError, match="add_loss_DA"):
            TrainStep(m, 4, 4, beta=BETA, add_loss_DA=bad)
    kw = dict(add_loss_DA="target_entropy")
    with pytest.raises(NotImplementedError, match="legacy"):
        TrainStep(m, 4, 4, beta=BETA, mode="phased", **kw)
    with pytest.raises(NotImplementedError, match="step program"):
        TrainStep(m, 4, 4, beta=BETA, class_weight=torch.ones(5), **kw)
    with pytest.raises(NotImplementedError, match="step program"):
        TrainStep(m, 4, 4, beta=BETA, domain_weight=(1.0, 0.5), **kw)
    with pytest.raises(NotImplementedError, match="step program"):
        TrainStep(m, 4, 4, beta=[-1.0, 0.75, 0.5], **kw)
    # the accepted values pass every check and stop at the device
    for ok in ("none", "attentive_entropy", "target_entropy"):
        with pytest.raises(Ta3nError, match="CUDA"):
            TrainStep(m, 4, 4, beta=BETA, add_loss_DA=ok)


def test_entry_validates_arguments():
    from ta3n_b200 import build
    build.build()
    from ta3n_b200 import _lib
    lib = _lib.load()
    assert lib.ta3n_target_entropy_fwd_bwd(None, 4, 7, 0.1, None, None, None, None, None) == 1
    assert b"ta3n_target_entropy_fwd_bwd" in lib.ta3n_last_error()
    assert lib.ta3n_target_entropy_fwd_bwd(16, 4, 0, 0.1, None, 32, 48, None, None) == 1          # C = 0
    assert lib.ta3n_target_entropy_fwd_bwd(16, -1, 7, 0.1, None, 32, 48, None, None) == 1         # rows < 0
    assert lib.ta3n_target_entropy_fwd_bwd(16, 4, 7, 0.1, None, 32, 16, None, None) == 1          # g_pred == pred
    assert b"alias" in lib.ta3n_last_error()
    assert lib.ta3n_target_entropy_fwd_bwd(None, 0, 7, 0.1, None, None, None, None, None) == 0    # empty target half


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------
def _dev():
    return torch.device("cuda:0")


def _model(T=5, C=7, drop=0.0, attn="TransAttn", attn_frame="none", ens="none", seed=3):
    from ta3n_b200.models import VideoModel
    torch.manual_seed(seed)
    m = VideoModel(C, "video", "trn-m", "RGB", train_segments=T, val_segments=T, fc_dim=256, dropout_i=drop,
                   dropout_v=drop, partial_bn=False, use_attn=attn, use_attn_frame=attn_frame, ens_DA=ens,
                   verbose=False)
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


STEP_CASES = {
    # name: (attn, attn_frame, ens, mu, drop, (Bs, Bt), (ns, nt), dis, gamma)
    "attn": ("TransAttn", "none", "none", 0.0, 0.0, (10, 7), (10, 7), None, 0.3),
    "attn_drop": ("TransAttn", "none", "none", 0.0, 0.5, (10, 7), (10, 7), None, 0.3),
    "none_drop": ("none", "none", "none", 0.0, 0.5, (8, 9), (8, 9), None, 0.3),
    "frame_attn_drop": ("TransAttn", "TransAttn", "none", 0.0, 0.5, (7, 9), (7, 9), None, 0.3),
    "mcd_mu0": ("TransAttn", "none", "MCD", 0.0, 0.0, (8, 6), (8, 6), None, 0.3),
    "mcd_mu07_drop": ("TransAttn", "none", "MCD", 0.7, 0.5, (8, 6), (8, 6), None, 0.3),
    "dan_drop": ("TransAttn", "none", "none", 0.0, 0.5, (10, 7), (10, 7), "DAN", 0.3),
    "short": ("TransAttn", "none", "none", 0.0, 0.5, (10, 7), (6, 4), None, 0.3),
    "mcd_short": ("TransAttn", "none", "MCD", 0.7, 0.5, (8, 6), (5, 2), None, 0.3),
}


@pytest.fixture(params=["fp32", "tf32x3", "tf32"])
def engine(request):
    import ta3n_b200
    ta3n_b200.set_gemm_engine(request.param)
    yield request.param
    ta3n_b200.set_gemm_engine("tf32x3")


def _entropy_logits(rows, C, seed):
    """randn * 3, with (where the rows exist) a large-spread row whose q underflows for half the classes and a
    uniform row (H = log C exactly, zero gradient)."""
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(rows, C, generator=g) * 3
    if rows > 1:
        z[rows // 2] = torch.where(torch.rand(C, generator=g) < 0.5, -80.0, 80.0) + torch.randn(C, generator=g)
    if rows > 2:
        z[rows - 1] = 2.5
    return z


def _entropy_ref(dt, z, vt, gamma, L0, G0, calls):
    """``calls`` launches from loss L0 and gradient G0: L0 + calls * gamma * term, G0 + calls * its gradient."""
    from tests.test_rowops_fp32 import _leaf
    p = _leaf(z, dt)
    term = teo.target_entropy(p[:vt])
    g = torch.autograd.grad(gamma * term, p)[0] if vt > 0 else torch.zeros_like(p)
    return dict(term=term.detach(), loss=torch.tensor(L0, dtype=dt) + calls * gamma * term.detach(),
                g=G0.to(dt) + calls * g)


@gpu
@pytest.mark.parametrize("C", [1, 7, 30, 32, 33, 1000])
@pytest.mark.parametrize("rows", [1, 31, 32, 33, 1024, 1500])
def test_entropy_entry_matches_fp64(rows, C):
    """ta3n_target_entropy_fwd_bwd alone against fp64 (test_rowops_fp32's rule, per row): rows past the 32 warps'
    first pass, classes past the lanes' first trip, valid_rows 0 / 1 / rows - 1 / rows / more than rows (clamped) and
    absent.  The loss, the gradient and the meter accumulate over two launches; padded rows keep their values bit for
    bit; a second run on fresh buffers gives the same bits."""
    from ta3n_b200._lib import check as lib_check
    from tests.test_rowops_fp32 import Buf, _guards, _lib, _ref, _st, check
    _, lib = _lib()
    gamma, L0, M0 = 0.7, 0.625, (3.5, -1.0, 11.0)
    z = _entropy_logits(rows, C, rows * 1009 + C)
    G0 = torch.randn(rows, C, generator=torch.Generator().manual_seed(C)) * 1e-3
    H = teo.target_entropy(z[rows - 1:].double()).item() if rows > 2 else None
    if H is not None:
        assert abs(H - np.log(C)) <= 1e-12 * max(1.0, np.log(C))
    for valid in sorted({0, 1, rows - 1, rows, rows + 5}) + [None]:
        vt = rows if valid is None else min(valid, rows)
        runs = []
        for _ in range(2):
            pb = Buf(rows, C, init=z.to(_dev()))
            loss = Buf(1, init=torch.full((1,), L0, device=_dev()))
            gp = Buf(rows, C, init=G0.to(_dev()))
            meter = torch.tensor(M0, device=_dev(), dtype=torch.float64)
            vr = None if valid is None else torch.tensor([17, valid], dtype=torch.int32, device=_dev())
            lib_check(lib.ta3n_target_entropy_fwd_bwd(pb.p, rows, C, gamma, None if vr is None else vr.data_ptr(),
                                                      loss.p, gp.p, meter.data_ptr(), _st()))
            torch.cuda.synchronize()
            runs.append((loss.cpu().clone(), gp.cpu().clone(), meter.cpu().clone()))
        assert all(torch.equal(a, b) for a, b in zip(*runs)), f"rows={rows} C={C} valid={valid}: reruns differ"
        what = f"rows={rows} C={C} valid={valid}"
        r64, r32 = _ref(_entropy_ref, z, vt, gamma, L0, G0, 1)
        q64 = torch.softmax(z.double(), 1)
        lq64 = torch.log_softmax(z.double(), 1)
        H64 = -(q64 * lq64).sum(1, keepdim=True)
        # the summands behind each gradient element: its start value and gamma/n * q (|log q| + H)
        scale = G0.double().abs() + gamma / max(vt, 1) * q64 * (lq64.abs() + H64)
        check(f"{what} term", runs[0][2][1], r64["term"], r32["term"], scale=torch.tensor(max(np.log(C), 1.0)))
        check(f"{what} loss", runs[0][0][0], r64["loss"], r32["loss"], scale=torch.tensor(L0 + gamma * np.log(C)))
        check(f"{what} g_pred", runs[0][1], r64["g"], r32["g"], dims=(0,), scale=scale)
        assert torch.equal(runs[0][1][vt:], G0[vt:]), f"{what}: a padded row's gradient changed"
        if C == 1:
            assert torch.equal(runs[0][1], G0) and runs[0][2][1].item() == 0.0
        if vt == 0:
            assert runs[0][0][0].item() == L0 and runs[0][2][1].item() == 0.0, f"{what}: no real row must add nothing"
        term = runs[0][2][1].item()
        assert runs[0][2][0].item() == M0[0] + term * vt and runs[0][2][2].item() == M0[2] + vt
        # a second launch on the same buffers: everything accumulates, the last value is the same bits
        vr = None if valid is None else torch.tensor([17, valid], dtype=torch.int32, device=_dev())
        lib_check(lib.ta3n_target_entropy_fwd_bwd(pb.p, rows, C, gamma, None if vr is None else vr.data_ptr(), loss.p,
                                                  gp.p, meter.data_ptr(), _st()))
        torch.cuda.synchronize()
        r64, r32 = _ref(_entropy_ref, z, vt, gamma, L0, G0, 2)
        check(f"{what} loss x2", loss.t[0], r64["loss"], r32["loss"], scale=torch.tensor(L0 + 2 * gamma * np.log(C)))
        check(f"{what} g_pred x2", gp.t, r64["g"], r32["g"], dims=(0,), scale=2 * scale)
        m = meter.cpu()
        assert m[1].item() == term and m[2].item() == M0[2] + 2 * vt
        assert m[0].item() == (M0[0] + term * vt) + term * vt
        assert torch.equal(gp.cpu()[vt:], G0[vt:])
        _guards(pb, loss, gp)
        assert torch.equal(pb.cpu(), z), "pred was written"


@gpu
@pytest.mark.parametrize("case", list(STEP_CASES))
def test_train_step_matches_fp64_oracle(case, engine):
    """One TrainStep against the fp64 oracle: loss, the term (loss_e meter) and every gradient; with dropout on, the
    oracle takes the masks rebuilt from the counter RNG with the step's seeds and the ReLU pattern the step realised
    (MCD: both passes', whose target logits differ, so the term must read pass 1's)."""
    from oracle import dropout_rng as drng
    from tests.pinned_pattern import realised_gates
    from tests.test_gpu_parity import FLIP_BOUND, NOISE_SCALE, PINNED_TOL, TOL
    from ta3n_b200.train import TrainStep
    attn, attn_frame, ens, mu, drop, (Bs, Bt), (ns, nt), dis, gamma = STEP_CASES[case]
    if dis and engine == "tf32":
        pytest.skip("the discrepancy suite runs DAN / JAN on the fp32 and tf32x3 engines only")
    T = 5
    m = _model(T=T, drop=drop, attn=attn, attn_frame=attn_frame, ens=ens)
    cfg = orc.PathConfig(num_class=7, num_segments=T, fc_dim=256, dropout_i=drop, dropout_v=drop, use_attn=attn,
                         use_attn_frame=attn_frame, ens_DA=ens)
    params = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    xs, xt, labels = _inputs(ns, nt, T)
    extra = dict(dis_DA=dis, alpha=0.7) if dis else {}
    step = TrainStep(m, Bs, Bt, BETA, gamma=gamma, use_graph=False, mu=mu, add_loss_DA="target_entropy", stats=True,
                     **extra)
    loss = step(xs.pin_memory(), xt.pin_memory(), labels)
    torch.cuda.synchronize()
    masks = masks2 = gates2 = None
    key = int(step.step_counter.item())
    if drop > 0:
        masks = drng.train_step_masks(key, Bs, Bt, T, cfg.shared_dim, cfg.video_dim, drop, drop, ns=ns, nt=nt)
        if ens == "MCD":
            masks2 = mcd.train_step_pass2_masks(key, Bt, T, cfg.shared_dim, cfg.video_dim, drop, drop, nt=nt)
    p64 = {k: v.double() if v.dtype.is_floating_point else v for k, v in params.items()}
    ones = lambda r: torch.ones(r, cfg.shared_dim, dtype=torch.bool)              # noqa: E731
    kept = ones((ns + nt) * T) if masks is None else torch.cat([masks["i_source"], masks["i_target"]]).bool()
    frames = lambda t: torch.cat([t[:ns * T], t[Bs * T:Bs * T + nt * T]]).cpu()    # noqa: E731
    videos = lambda t: torch.cat([t[:ns], t[Bs:Bs + nt]]).cpu()                    # noqa: E731
    plain = orc.activation_pattern(p64, xs.double(), xt.double(), BETA, cfg, masks=masks)
    gates, flips, total = realised_gates(step.bufs.pool, frames, videos, kept, plain, True, True)
    if ens == "MCD":
        k2 = None if masks2 is None else {"i_source": torch.ones(0, cfg.shared_dim, dtype=torch.uint8),
                                          "v_source": torch.ones(0, cfg.video_dim, dtype=torch.uint8), **masks2}
        plain2 = orc.activation_pattern(p64, xs[:0].double(), xt.double(), BETA, cfg, masks=k2)
        kept2 = ones(nt * T) if masks2 is None else masks2["i_target"].bool()
        g2, f2, n2 = realised_gates(step.bufs2.pool, lambda t: t[:nt * T].cpu(), lambda t: t[:nt].cpu(), kept2,
                                    plain2, attn_frame != "none", False)
        _, gates2 = orc.split_gates(g2, 0, T)
        flips, total = flips + f2, total + n2
    assert flips <= max(FLIP_BOUND[engine] * total, 2), (flips, total)
    kw = dict(train=drop > 0, masks=masks, gates=gates, mu=mu, masks2=masks2, gates2=gates2, dis_DA=dis, alpha=0.7)
    l64, t64, g64 = teo.entropy_train_step(p64, xs.double(), xt.double(), labels, BETA, cfg, gamma, **kw)
    _, t32, g32 = teo.entropy_train_step(params, xs, xt, labels, BETA, cfg, gamma, **kw)
    assert_close(loss.cpu()[0], l64, TOL[engine], "loss")
    st = step.stats()
    assert st.loss_e.count == nt
    assert_close(torch.tensor(st.loss_e.val), t64, TOL[engine], "term", noise=abs(t32.double() - t64).item() * 8)
    named = dict(m.named_parameters())
    for name, g in g64.items():
        if g is None:
            continue
        noise = (g32[name].double() - g).norm().item() * NOISE_SCALE[engine]
        assert_close(named[name].grad, g, PINNED_TOL[engine], f"grad {name}", noise=noise)


@gpu
def test_batch_without_target_rows_equals_the_step_without_the_term():
    """No real target row: the term adds nothing, bit for bit."""
    from ta3n_b200.train import TrainStep
    xs, xt, labels = _inputs(6, 4, 5)
    m_a = _model(drop=0.5)
    m_b = copy.deepcopy(m_a)
    plain = TrainStep(m_a, 6, 4, BETA, seed=3, add_loss_DA="none")
    step = TrainStep(m_b, 6, 4, BETA, seed=3, add_loss_DA="target_entropy")
    la, lb = plain(xs, xt[:0], labels).clone(), step(xs, xt[:0], labels).clone()
    torch.cuda.synchronize()
    assert torch.equal(la, lb)
    assert torch.equal(plain.flat_grad, step.flat_grad)


@gpu
@pytest.mark.parametrize("ens", ["none", "MCD"])
def test_eager_graph_and_reruns_are_bit_identical(ens):
    """Eager == graph, and a second run == the first, bit for bit over three SGD steps (dropout on, a short batch
    among them)."""
    from ta3n_b200.train import SGDNesterov, TrainStep
    xs, xt, labels = _inputs(8, 6, 5)
    runs = []
    for use_graph in (False, True, True):
        m = _model(drop=0.5, ens=ens)
        step = TrainStep(m, 8, 6, BETA, use_graph=use_graph, optimizer=SGDNesterov(lr=0.01), seed=11, gamma=0.3,
                         add_loss_DA="target_entropy", mu=0.7 if ens == "MCD" else 0.0)
        if use_graph:
            step.step_counter.fill_(0)       # the capture's warm-up advanced the dropout counter
        losses = []
        for i in range(3):
            n = (8, 6) if i != 1 else (5, 3)
            losses.append(step(xs[:n[0]], xt[:n[1]], labels[:n[0]]).clone())
        torch.cuda.synchronize()
        runs.append((torch.cat(losses), step.flat_param.clone()))
    for other in runs[1:]:
        assert torch.equal(runs[0][0], other[0]) and torch.equal(runs[0][1], other[1])


@gpu
@pytest.mark.parametrize("attn", ["TransAttn", "none"])
def test_three_steps_match_the_stock_autograd_loop(attn):
    """Three SGDNesterov steps against main.py's loop on this repo's VideoModel: autograd, clip_grad_norm_ and
    torch.optim.SGD(nesterov=True), with ta3n_loss(..., add_loss_DA='target_entropy')."""
    import ta3n_b200
    from ta3n_b200 import loss as LS
    from ta3n_b200.train import SGDNesterov, TrainStep
    ta3n_b200.set_gemm_engine("fp32")
    try:
        xs, xt, labels = _inputs(8, 6, 5)
        m_a = _model(attn=attn)
        m_b = copy.deepcopy(m_a)
        step = TrainStep(m_a, 8, 6, BETA, gamma=0.3, optimizer=SGDNesterov(lr=0.01, clip_gradient=0.5),
                         add_loss_DA="target_entropy")
        for _ in range(3):
            step(xs, xt, labels)
        torch.cuda.synchronize()
        params = list(m_b.parameters())
        opt = torch.optim.SGD(params, 0.01, momentum=0.9, weight_decay=1e-4, nesterov=True)
        d = _dev()
        for _ in range(3):
            opt.zero_grad(set_to_none=True)
            outs = m_b(xs.to(d), xt.to(d), list(BETA), 0, is_train=True, reverse=False)
            loss = LS.ta3n_loss(outs, labels.to(d), 0.3, use_attn=attn, add_loss_DA="target_entropy")
            loss.backward()
            torch.nn.utils.clip_grad_norm_([p for p in params if p.grad is not None], 0.5)
            opt.step()
        pb = dict(m_b.named_parameters())
        for name, p in m_a.named_parameters():
            assert_close(p.detach(), pb[name].detach(), 1e-5, name)
    finally:
        ta3n_b200.set_gemm_engine("tf32x3")


@gpu
def test_resume_from_state_dict_is_bit_identical():
    from ta3n_b200.train import SGDNesterov, TrainStep
    xs, xt, labels = _inputs(6, 5, 5)
    m_a = _model(drop=0.5, ens="MCD")
    m_b = copy.deepcopy(m_a)
    kw = dict(optimizer=SGDNesterov(lr=0.01), seed=5, add_loss_DA="target_entropy", gamma=0.3, mu=0.7)
    a = TrainStep(m_a, 6, 5, BETA, **kw)
    for _ in range(4):
        a(xs, xt, labels)
    b0 = TrainStep(m_b, 6, 5, BETA, **kw)
    for _ in range(2):
        b0(xs, xt, labels)
    sd = copy.deepcopy(b0.state_dict())
    params = copy.deepcopy(m_b.state_dict())
    m_c = _model(drop=0.5, ens="MCD", seed=99)
    m_c.load_state_dict(params)
    c = TrainStep(m_c, 6, 5, BETA, **kw)
    c.load_state_dict(sd)
    for _ in range(2):
        c(xs, xt, labels)
    torch.cuda.synchronize()
    assert torch.equal(a.flat_param, c.flat_param)


@gpu
def test_meters_equal_the_reference_average_meters():
    """Over an epoch with a short last batch and a batch without target rows, stats() / stats_async() against
    AverageMeters fed as main.py feeds them: losses_e with loss.py's cross_entropy_soft of the real target rows'
    logits (computed here in fp64 from the logits the step produced) and n = those rows (main.py:544; a batch without
    target rows adds n = 0), the loss meter with the loss the step reports (losses.update(loss.item()), n = 1)."""
    from oracle.train_stats_oracle import AverageMeter
    from ta3n_b200.train import TrainStep
    Bs = 8
    xs, xt, labels = _inputs(Bs, 6, 5)
    step = TrainStep(_model(drop=0.5), Bs, 6, BETA, gamma=0.3, add_loss_DA="target_entropy", stats=True)
    ref_e, ref_l = AverageMeter(), AverageMeter()
    for ns, nt in ((8, 6), (8, 6), (8, 0), (5, 2)):
        loss = step(xs[:ns], xt[:nt], labels[:ns]).item()
        logits_t = step.outputs[5][Bs:Bs + nt].double().cpu()
        ref_e.update(teo.target_entropy(logits_t).item(), nt)
        ref_l.update(loss)
    st, snap = step.stats(), step.stats_async().result()
    for got in (st, snap):
        assert got.loss_e.count == ref_e.count == 14
        assert got.loss_e.val == pytest.approx(ref_e.val, rel=1e-5)
        assert got.loss_e.sum == pytest.approx(ref_e.sum, rel=1e-5)
        assert got.loss_e.avg == pytest.approx(ref_e.avg, rel=1e-5)
        assert got.loss.avg == pytest.approx(ref_l.avg, rel=1e-6) and got.loss.count == 4
    step.reset_stats()
    assert step.stats().loss_e.count == 0


@gpu
def test_meter_term_equals_the_oracle_on_the_logits():
    """The loss_e meter's value is the entropy of the step's own target logits, and the loss includes gamma times
    it: the loss minus the same step without the term."""
    from ta3n_b200.train import TrainStep
    xs, xt, labels = _inputs(8, 6, 5)
    m_a = _model()
    m_b = copy.deepcopy(m_a)
    plain = TrainStep(m_a, 8, 6, BETA, gamma=0.3, add_loss_DA="none")
    step = TrainStep(m_b, 8, 6, BETA, gamma=0.3, add_loss_DA="target_entropy", stats=True)
    l0, l1 = plain(xs, xt, labels).item(), step(xs, xt, labels).item()
    torch.cuda.synchronize()
    term = teo.target_entropy(step.outputs[5][8:].double().cpu()).item()
    assert step.stats().loss_e.val == pytest.approx(term, rel=1e-5)
    assert l1 - l0 == pytest.approx(0.3 * term, rel=1e-4, abs=1e-6)


@gpu
@pytest.mark.parametrize("with_opt", [False, True])
def test_launches_the_term_adds(with_opt):
    """The default step (attentive entropy) issues the launches it did before this option existed; the target entropy
    adds one launch to the step without an entropy term."""
    import ta3n_b200
    from tests.test_discrepancy import PLAIN_LAUNCHES
    from ta3n_b200.train import SGDNesterov, TrainStep
    ta3n_b200.set_gemm_engine("tf32x3")
    counts = {}
    for mode in ("attentive_entropy", "none", "target_entropy"):
        step = TrainStep(_model(), 8, 6, BETA, add_loss_DA=mode,
                         optimizer=SGDNesterov(lr=0.01) if with_opt else None)
        counts[mode] = step.launches_per_step
    assert counts["attentive_entropy"] == PLAIN_LAUNCHES[with_opt], counts
    assert counts["none"] == counts["attentive_entropy"], counts
    assert counts["target_entropy"] == counts["none"] + 1, counts


@gpu
@pytest.mark.parametrize("ens", ["none", "MCD"])
def test_train_step_from_device_sampler_is_bit_identical_to_load(tmp_path, ens):
    """TrainStep(add_loss_DA='target_entropy') fed by the device sampler against the same step fed the same batches
    through load(), seeded alike, over two epochs with short last batches on both sides: loss, parameters and momentum
    equal bit for bit after every step."""
    from ta3n_b200 import dataset as D
    from ta3n_b200.train import SGDNesterov, TrainStep
    from tests.test_device_sampler import _banks
    T, batch = 5, (8, 6)
    sets, banks = _banks(tmp_path, T, orc.FEATURE_DIM, (21, None), (9, 14), batch)     # 3 iterations, ends 5 + 2
    model_a = _model(drop=0.5, ens=ens)
    model_b = copy.deepcopy(model_a)
    kw = dict(beta=BETA, gamma=0.3, seed=123, add_loss_DA="target_entropy", mu=0.7 if ens == "MCD" else 0.0)
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
            assert torch.equal(step_a.valid, step_b.valid)
            assert torch.equal(loss_a, loss_b), (epoch, n_step, loss_a.item(), loss_b.item())
            assert torch.equal(step_a.flat_param, step_b.flat_param), (epoch, n_step)
            assert torch.equal(step_a.momentum_buf, step_b.momentum_buf), (epoch, n_step)
    assert n_step == 6
