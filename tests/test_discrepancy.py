"""Discrepancy-based alignment (--dis_DA DAN / JAN): multi-kernel MMD and JAN as CUDA loss kernels in TrainStep.

CPU: loss.mmd_rbf / JAN / discrepancy_loss and the fp64 oracle (oracle/dis_oracle.py) against the reference's values
(tests/golden/dis_golden.npz), the options TrainStep refuses, the C ABI's argument checks.
GPU: the kernels against fp64 at fp32 grade (per row of the gradient), guards, NaN and zero cases, bit-identical
reruns; TrainStep against the fp64 oracle, eager == graph, set_alpha without re-capture, SGD / Adam against
torch.optim, resume, the meters, and the launches the term adds.
"""
import copy
import json
import os

import numpy as np
import pytest
import torch

from oracle import dis_oracle as dor
from oracle import gen_golden_dis as gen
from tests.golden_util import TOL_FP32, assert_close

gpu = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
BETA = (0.75, 0.6, 0.5)


def _golden():
    z = np.load(os.path.join(HERE, "golden", "dis_golden.npz"))
    return z, json.loads(bytes(z["meta_json"]).decode())


def _assert_stored(t, z, key, tol, what, noise=0.0):
    t = t.detach().double().cpu()
    if key in z.files:
        assert tuple(t.shape) == z[key].shape, (what, tuple(t.shape), z[key].shape)
        assert_close(t, z[key], tol, what, noise=noise)
        return
    _, n = z[key + "#stats"]
    flat = t.reshape(-1)
    assert abs(flat.norm().item() - n) <= tol * n + 8 * noise, f"{what}: norm {flat.norm().item():.6e} vs {n:.6e}"
    assert_close(flat[::gen.STRIDE], z[key + "#sample"], tol * 4, what + " (sample)", noise=noise)


def _cpu_model(**kw):
    from ta3n_b200.models import VideoModel
    args = dict(train_segments=5, val_segments=5, fc_dim=64, verbose=False)
    args.update(kw)
    return VideoModel(5, "video", "trn-m", "RGB", **args).train()


def _case_params(c, order):
    """The reference's initial parameters of a golden case (this package's VideoModel seeds them identically), moved
    as the generator moves them."""
    from ta3n_b200.models import VideoModel
    torch.manual_seed(gen.MODEL_SEED)
    m = VideoModel(c["C"], "video", "trn-m", "RGB", train_segments=c["T"], val_segments=c["T"], add_fc=c["add_fc"],
                   fc_dim=c["F"], dropout_i=c["drop"], dropout_v=c["drop"], partial_bn=False, ens_DA=c["ens"],
                   use_attn=c["use_attn"], verbose=False)
    named = {k: v.detach().clone() for k, v in m.named_parameters()}
    gen.perturb(named, order)
    return named, m


# ---- CPU: the torch ops and the oracle against the reference ------------------------------------------------------
@pytest.mark.parametrize("n", gen.ALONE_N)
@pytest.mark.parametrize("d", gen.ALONE_D)
def test_loss_functions_equal_the_reference(n, d):
    """loss.mmd_rbf (kernel_num 2 and 5) and loss.JAN: value and input gradients against the reference's."""
    from ta3n_b200 import loss as LS
    z, _ = _golden()
    xs, xt, ys, yt = [t.requires_grad_(True) for t in gen.alone_inputs(n, d)]
    fns = {"mmd2": lambda: LS.mmd_rbf(xs, xt, kernel_mul=2.0, kernel_num=2),
           "mmd5": lambda: LS.mmd_rbf(xs, xt, kernel_mul=2.0, kernel_num=5),
           "jan": lambda: LS.JAN([ys, xs], [yt, xt], kernel_muls=[2.0, 2.0], kernel_nums=[2, 5])}
    for name, fn in fns.items():
        k = f"alone/{name}/n{n}_d{d}/"
        val = fn()
        grads = torch.autograd.grad(val, [xs, xt, ys, yt], allow_unused=True)
        assert_close(val.detach(), z[k + "value"], TOL_FP32, k + "value", noise=float(z[k + "noise/value"]))
        for gname, g in zip(("xs", "xt", "ys", "yt"), grads):
            if g is None:
                assert k + "grad_noise/" + gname not in z.files
                continue
            _assert_stored(g, z, k + "grad/" + gname, TOL_FP32, k + gname,
                           noise=max(float(z[k + "grad_noise/" + gname]), 1e-12))


def test_loss_ver1_and_gaussian_kernel():
    """ver=1 (the linear-time estimate) and guassian_kernel with a fixed sigma, against a direct restatement."""
    from ta3n_b200 import loss as LS
    g = torch.Generator().manual_seed(3)
    xs, xt = torch.randn(6, 4, generator=g, dtype=torch.float64), torch.randn(6, 4, generator=g, dtype=torch.float64)
    k = LS.guassian_kernel(xs, xt, kernel_mul=2.0, kernel_num=3, fix_sigma=1.5)
    rows = torch.cat([xs, xt])
    l2 = torch.cdist(rows, rows) ** 2
    want = sum(torch.exp(-l2 / (1.5 / 2.0 * 2.0 ** i)) for i in range(3))
    assert torch.allclose(k, want, rtol=1e-12, atol=1e-12)
    kk = LS.guassian_kernel(xs, xt, 2.0, 5)
    v1 = sum(kk[i, (i + 1) % 6] + kk[i + 6, (i + 1) % 6 + 6] - kk[i, (i + 1) % 6 + 6] - kk[(i + 1) % 6, i + 6]
             for i in range(6))
    assert LS.mmd_rbf(xs, xt, ver=1).item() == pytest.approx(abs(v1.item()) / 6, rel=1e-12)
    with pytest.raises(ValueError):
        LS.mmd_rbf(xs, xt, ver=3)


@pytest.mark.parametrize("case", list(gen.CASES))
def test_oracle_iteration_equals_golden(case):
    """The fp64 oracle of the iteration (loss, loss_d, every gradient) against the reference's, and
    loss.discrepancy_loss on the oracle's fp32 outputs against the reference's loss_d."""
    from oracle import add_fc_oracle as afo
    from ta3n_b200 import loss as LS
    z, meta = _golden()
    k = case + "/"
    c = gen.CASES[case]
    params, _ = _case_params(c, meta[k + "param_order"])
    cfg, xs, xt, labels, m1, m2 = gen.case_inputs(c)
    p64 = {n: v.double() for n, v in params.items()}
    loss, loss_d, grads = dor.dis_train_step(p64, xs.double(), xt.double(), labels, BETA, cfg, c["dis"], c["alpha"],
                                             c["place"], add_fc=c["add_fc"], gamma=gen.GAMMA, train=c["drop"] > 0,
                                             masks=m1, mu=c["mu"], masks2=m2)
    assert_close(loss, z[k + "loss"], TOL_FP32, f"{case} loss", noise=float(z[k + "noise/loss"]))
    assert_close(loss_d, z[k + "loss_d"], TOL_FP32, f"{case} loss_d", noise=float(z[k + "noise/loss_d"]))
    with_grad = meta[k + "with_grad"]
    assert sorted(n for n, g in grads.items() if g is not None) == sorted(with_grad)
    for n in with_grad:
        _assert_stored(grads[n], z, k + "grad/" + n, 2e-4, f"{case} grad {n}",
                       noise=max(float(z[k + "grad_noise/" + n]), 4e-9))
    # the package's torch op on the oracle's fp32 forward (pass 1 of MCD is the plain forward)
    with torch.no_grad():
        o = afo.forward(params, xs, xt, BETA, 0.0, cfg, c["add_fc"], train=c["drop"] > 0,
                        masks={kk: v for kk, v in (m1 or {}).items()})
        got = LS.discrepancy_loss(list(o[4]), list(o[9]), c["dis"], c["add_fc"], tuple(c["place"]))
    assert_close(got, z[k + "loss_d"], 2e-4, f"{case} discrepancy_loss", noise=float(z[k + "noise/loss_d"]))


def test_discrepancy_loss_degenerate_and_refused_inputs():
    from ta3n_b200 import loss as LS
    g = torch.Generator().manual_seed(1)
    fs = [torch.randn(5, 3, generator=g), torch.randn(5, 8, generator=g), torch.randn(5, 4, 6, generator=g)]
    ft = [t[:0] for t in fs]
    assert LS.discrepancy_loss(fs, ft, "DAN").item() == 0.0           # no target row
    assert LS.discrepancy_loss(fs, ft, "JAN").item() == 0.0
    big = [torch.randn(300, 3, generator=g), torch.randn(300, 8, generator=g)]
    assert LS.discrepancy_loss(big, big, "DAN").item() == 0.0         # 300 rows: the reference's view() fails
    same = [torch.ones(4, 3), torch.ones(4, 8)]
    assert torch.isnan(LS.discrepancy_loss(same, same, "DAN", place_dis="YNN"))       # bandwidth 0, as the reference
    with pytest.raises(NotImplementedError):
        LS.discrepancy_loss(fs, fs, "CORAL")
    with pytest.raises(ValueError):
        LS.discrepancy_loss(fs, fs, "MMD")
    with pytest.raises(ValueError, match="3-D"):
        LS.discrepancy_loss(fs, fs, "DAN", place_dis="YYY")
    with pytest.raises(ValueError, match="entries"):
        LS.discrepancy_loss(fs, fs, "DAN", add_fc=2, place_dis="YYN")
    with pytest.raises(ValueError, match="no level"):
        LS.discrepancy_loss(fs, fs, "DAN", place_dis="NNN")


def test_train_step_discrepancy_refusals():
    from ta3n_b200 import Ta3nError
    from ta3n_b200.train import TrainStep, alpha_dann
    m = _cpu_model()
    with pytest.raises(NotImplementedError, match="legacy"):
        TrainStep(m, 4, 4, beta=BETA, dis_DA="DAN", mode="phased")
    with pytest.raises(NotImplementedError, match="step program"):
        TrainStep(m, 4, 4, beta=BETA, dis_DA="DAN", class_weight=torch.ones(5))
    with pytest.raises(NotImplementedError, match="step program"):
        TrainStep(m, 4, 4, beta=[-1.0, 0.75, 0.5], dis_DA="JAN")
    with pytest.raises(NotImplementedError, match="step program"):
        TrainStep(m, 4, 4, beta=BETA, dis_DA="JAN", domain_weight=(1.0, 2.0))
    with pytest.raises(NotImplementedError, match="CORAL"):
        TrainStep(m, 4, 4, beta=BETA, dis_DA="CORAL")
    with pytest.raises(ValueError, match="dis_DA"):
        TrainStep(m, 4, 4, beta=BETA, dis_DA="MMD")
    with pytest.raises(ValueError, match="3-D"):
        TrainStep(m, 4, 4, beta=BETA, dis_DA="DAN", place_dis=("Y", "Y", "Y"))
    with pytest.raises(ValueError, match="entries"):
        TrainStep(_cpu_model(add_fc=2), 4, 4, beta=BETA, dis_DA="DAN", place_dis=("Y", "Y", "N"))
    with pytest.raises(ValueError, match="256"):
        TrainStep(m, 300, 320, beta=BETA, dis_DA="DAN")
    with pytest.raises(ValueError, match="alpha"):
        TrainStep(m, 4, 4, beta=BETA, alpha=0.5)
    for dis in ("DAN", "JAN"):                  # main.py:231: a negative --alpha means the schedule, not a weight
        with pytest.raises(ValueError, match="alpha_dann"):
            TrainStep(m, 4, 4, beta=BETA, dis_DA=dis, alpha=-1.0)
    with pytest.raises(ValueError, match="no level"):
        TrainStep(m, 4, 4, beta=BETA, dis_DA="DAN", place_dis=("N", "N", "N"))
    # what passes these checks stops at the device: JAN ignores place_dis, DAN at 512 rows cuts two chunks
    for kw in (dict(dis_DA="JAN", place_dis=("Y", "Y", "Y")), dict(dis_DA="JAN", place_dis=("N", "N", "N")),
               dict(dis_DA="DAN", alpha=0.5), dict(dis_DA="DAN", place_dis=("N", "Y", "N", "N"))):
        with pytest.raises(Ta3nError, match="CUDA"):
            TrainStep(_cpu_model(add_fc=2) if len(kw.get("place_dis", "")) == 4 else m, 4, 4, beta=BETA, **kw)
    with pytest.raises(Ta3nError, match="CUDA"):
        TrainStep(m, 512, 600, beta=BETA, dis_DA="DAN")
    assert alpha_dann(0, 10) == 0.0
    assert alpha_dann(10, 10) == pytest.approx(2 / (1 + np.exp(-1.0)) - 1, rel=1e-15)
    assert alpha_dann(7, 10) == pytest.approx(dor.alpha_dann(7, 10), rel=1e-15)


def test_train_step_discrepancy_refuses_several_ranks(monkeypatch):
    import torch.distributed as dist
    from ta3n_b200.train import TrainStep
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    with pytest.raises(NotImplementedError, match="single rank"):
        TrainStep(_cpu_model(), 4, 4, beta=BETA, dis_DA="DAN")


def test_train_stats_gains_an_empty_loss_d_meter():
    from ta3n_b200.train import Meter, dis_meter, parse_train_stats
    st = parse_train_stats(np.zeros(27, dtype=np.int64), (1, 5))
    assert st.loss_d == Meter()
    assert dis_meter([3.0, 0.5, 6.0]) == Meter(val=0.5, avg=0.5, sum=3.0, count=6)


def test_discrepancy_entry_validates_arguments():
    from ta3n_b200 import _lib
    lib = _lib.load()
    assert lib.ta3n_discrepancy_workspace_bytes(0, 4, 0) == 0
    assert lib.ta3n_discrepancy_workspace_bytes(300, 600, 0) >= 2 * (512 * 512) * 4     # one 256-row chunk
    assert lib.ta3n_discrepancy_workspace_bytes(600, 600, 0) >= 2 * 2 * (512 * 512) * 4
    assert lib.ta3n_discrepancy_workspace_bytes(300, 600, 1) >= 2 * (600 * 600) * 4
    none = [None, None, 0, 0, 0.0, None, None]
    args = dict(store=0, valid=None, alpha=None, loss=16, loss_d=32, meter=None, ws=64, nbytes=1 << 30)

    def call(joint, l0, l1, **kw):
        a = {**args, **kw}
        return lib.ta3n_discrepancy_fwd_bwd(joint, 4, 4, *l0, *l1, a["store"], a["valid"], a["alpha"], a["loss"],
                                            a["loss_d"], a["meter"], a["ws"], a["nbytes"], None)
    assert call(0, none, none) == 1 and b"no layer" in lib.ta3n_last_error()
    assert call(0, [16, 32, 8, 2, 2.0, None, 48], none) == 1
    assert call(0, [16, 32, 8, 0, 2.0, 64, 48], none) == 1
    assert call(0, [16, 32, 8, 2, 2.0, 16, 48], none) == 1 and b"alias" in lib.ta3n_last_error()
    assert call(0, [16, 32, 8, 2, 2.0, 64, 48], none, nbytes=16) == 1 and b"workspace" in lib.ta3n_last_error()
    assert call(0, [16, 32, 8, 2, 2.0, 64, 48], none, loss=None) == 1


# ---- GPU: the kernels against fp64 --------------------------------------------------------------------------------
def _dev():
    return torch.device("cuda:0")


def _ref_term(srcs, tgts, joint, nums, n, dtype):
    """The term and its input gradients in ``dtype`` on the CPU: joint = one chunk of n rows with the product kernel;
    else each layer a DAN level over chunks of min(256, n) rows (0 when 256 does not divide n > 256)."""
    xs = [s[:n].detach().cpu().to(dtype).requires_grad_(True) for s in srcs]
    xt = [t[:n].detach().cpu().to(dtype).requires_grad_(True) for t in tgts]
    if n == 0 or (not joint and n > 256 and n % 256):
        return torch.zeros((), dtype=dtype), [torch.zeros_like(x) for x in xs + xt]
    if joint:
        k = None
        for i in range(len(xs)):
            kl = dor.kernel_sum(torch.cat([xs[i], xt[i]]), nums[i])
            k = kl if k is None else k * kl
        val = dor.mmd(k, n)
    else:
        s = min(256, n)
        val = 0
        for i in range(len(xs)):
            parts = [dor.mmd(dor.kernel_sum(torch.cat([xs[i][c:c + s], xt[i][c:c + s]]), nums[i]), s)
                     for c in range(0, n, s)]
            val = val + sum(parts) / len(parts)
    grads = torch.autograd.grad(val, xs + xt)
    return val.detach(), list(grads)


def _check_rows(got, r64, r32, what, start=None):
    """Per row: ||got - ref64|| <= TOL_FP32 ||ref64|| + 8 ||ref32 - ref64|| (tests/test_rowops_fp32.py's rule).
    ``start``: the values the kernel added to; the sum's own fp32 rounding (half an ulp per element) is allowed."""
    got = got.detach().double().cpu()
    bound = TOL_FP32 * r64.norm(dim=1) + 8 * (r32.double() - r64).norm(dim=1)
    if start is not None:
        r64 = r64 + start.detach().double().cpu()
        bound = bound + 2.0 ** -24 * r64.norm(dim=1)
    d = (got - r64).norm(dim=1)
    bad = (d > bound) & ~((d == 0) & (bound == 0))
    assert not bad.any(), f"{what}: rows {bad.nonzero().flatten()[:8].tolist()} err {d[bad][:4].tolist()} " \
                          f"bound {bound[bad][:4].tolist()}"


GUARD = 3


def _guarded(rows, d, fill, gen_):
    """A [rows, d] view inside a buffer with GUARD NaN rows on each side; ``fill``: 'rand' or 'nan'."""
    buf = torch.full((rows + 2 * GUARD, d), float("nan"), device=_dev())
    view = buf[GUARD:GUARD + rows]
    if fill == "rand":
        view.copy_(torch.randn(rows, d, generator=gen_).to(_dev()))
    return buf, view


KERNEL_CASES = [
    # (joint, widths, capacity (Bs, Bt), real rows (vs, vt), alpha)
    (False, (5,), (1, 3), (1, 3), 1.0),
    (False, (12, 1000), (2, 2), (2, 2), 0.3),
    (False, (1000,), (40, 45), (37, 41), 1.0),
    (False, (10, 256), (256, 300), (256, 300), 0.3),
    (False, (12, 512), (512, 512), (512, 512), 1.0),          # two chunks per level
    (False, (1024,), (600, 520), (512, 530), 0.0),
    (True, (5, 12), (1, 1), (1, 1), 1.0),
    (True, (12, 256), (40, 37), (39, 37), 0.3),
    (True, (5, 1024), (300, 310), (300, 305), 1.0),
    (True, (1000, 512), (256, 256), (256, 256), 1.0),
    (True, (256,), (520, 512), (512, 512), 1.0),              # one layer alone: mmd_rbf over 512 rows, no chunks
]


def _run_kernel(joint, widths, cap, real, alpha, store, seed=0):
    from ta3n_b200 import _lib
    from ta3n_b200 import functional as TF
    g = torch.Generator().manual_seed(seed)
    Bs, Bt = cap
    srcs = [torch.randn(Bs, d, generator=g).to(_dev()) for d in widths]
    tgts = [(torch.randn(Bt, d, generator=g) * 1.3 + 0.2).to(_dev()) for d in widths]
    nums = (5,) if len(widths) == 1 else (2, 5)
    grads = []
    layers = [None, None]
    slot = (1,) if len(widths) == 1 else (0, 1)
    for i, d in enumerate(widths):
        bs_, gs = _guarded(Bs, d, "rand", g)
        bt_, gt = _guarded(Bt, d, "rand", g)
        grads.append((bs_, gs, gs.clone(), bt_, gt, gt.clone()))
        layers[slot[i]] = (srcs[i], tgts[i], gs, gt, nums[i], 2.0)
    valid = torch.tensor(real, dtype=torch.int32, device=_dev())
    alpha_t = torch.tensor([alpha], device=_dev())
    loss = torch.full((1,), 0.25, device=_dev())
    loss_d = torch.full((1,), 7.0, device=_dev())
    ws = torch.empty(_lib.load().ta3n_discrepancy_workspace_bytes(Bs, Bt, int(joint)), dtype=torch.uint8, device=_dev())
    ws.fill_(0xFF)                                      # NaN bit patterns: every value the kernels read is written first
    meter = torch.zeros(3, dtype=torch.float64, device=_dev())
    TF.discrepancy_fwd_bwd(joint, layers, Bs, Bt, valid, alpha_t, loss, loss_d, ws,
                           store=sum(1 << s for s in slot) if store else 0, meter=meter)
    torch.cuda.synchronize()
    return srcs, tgts, nums, grads, loss, loss_d, meter


@gpu
@pytest.mark.parametrize("store", [False, True])
@pytest.mark.parametrize("case", range(len(KERNEL_CASES)))
def test_kernels_match_fp64(case, store):
    joint, widths, cap, real, alpha = KERNEL_CASES[case]
    srcs, tgts, nums, grads, loss, loss_d, meter = _run_kernel(joint, widths, cap, real, alpha, store, seed=case)
    n = min(real)
    v64, g64 = _ref_term(srcs, tgts, joint, nums, n, torch.float64)
    v32, g32 = _ref_term(srcs, tgts, joint, nums, n, torch.float32)
    what = f"joint={joint} widths={widths} cap={cap} real={real} alpha={alpha} store={store}"
    assert_close(loss_d.cpu()[0], v64, TOL_FP32, what + " loss_d", noise=abs(v32.double() - v64).item())
    assert_close(loss.cpu()[0] - 0.25, alpha * v64, 4e-5, what + " loss", noise=alpha * abs(v32.double() - v64).item())
    assert meter.cpu().tolist() == [float(loss_d.cpu()[0]) * real[0], float(loss_d.cpu()[0]), float(real[0])]
    k = len(widths)
    for i in range(k):
        bs_, gs, gs0, bt_, gt, gt0 = grads[i]
        for buf in (bs_, bt_):                                          # guards untouched
            assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[-GUARD:]).all(), what
        for view, start, ref64, ref32, cap_rows in ((gs, gs0, g64[i], g32[i], cap[0]), (gt, gt0, g64[k + i],
                                                                                         g32[k + i], cap[1])):
            _check_rows(view[:n], alpha * ref64, alpha * ref32.double(), f"{what} layer {i}",
                        start=None if store else start[:n])
            rest = view[n:cap_rows]
            assert torch.equal(rest, torch.zeros_like(rest) if store else start[n:cap_rows]), what


@gpu
def test_kernels_degenerate_and_empty_batches():
    """A chunk of identical rows gives NaN as the reference does; no real target row, or a DAN batch of more than 256
    rows that 256 does not divide, adds exactly 0 to the loss and the gradient."""
    from ta3n_b200 import loss as LS
    from ta3n_b200 import functional as TF
    x = torch.ones(4, 6, device=_dev())
    v = TF.mmd_loss(x, x.clone(), 2.0, 5)
    assert torch.isnan(v) and torch.isnan(LS.mmd_rbf(x.cpu(), x.cpu()))
    for joint, cap, real in ((False, (8, 8), (8, 0)), (True, (8, 8), (5, 0)), (False, (512, 512), (300, 512))):
        _, _, _, grads, loss, loss_d, meter = _run_kernel(joint, (7, 20), cap, real, 1.0, False)
        assert loss.item() == 0.25 and loss_d.item() == 0.0
        assert meter.cpu().tolist() == [0.0, 0.0, float(real[0])]
        for bs_, gs, gs0, bt_, gt, gt0 in grads:
            assert torch.equal(gs, gs0) and torch.equal(gt, gt0)
        _, _, _, grads, _, _, _ = _run_kernel(joint, (7, 20), cap, real, 1.0, True)
        for bs_, gs, gs0, bt_, gt, gt0 in grads:
            assert not gs.any() and not gt.any()


@gpu
@pytest.mark.parametrize("case", [1, 4, 8])
def test_kernels_rerun_bit_identical(case):
    joint, widths, cap, real, alpha = KERNEL_CASES[case]
    a = _run_kernel(joint, widths, cap, real, alpha, True, seed=7)
    b = _run_kernel(joint, widths, cap, real, alpha, True, seed=7)
    assert torch.equal(a[4], b[4]) and torch.equal(a[5], b[5])
    for ga, gb in zip(a[3], b[3]):
        assert torch.equal(ga[1], gb[1]) and torch.equal(ga[4], gb[4])


@gpu
def test_autograd_wrappers_match_the_torch_ops():
    from ta3n_b200 import functional as TF
    from ta3n_b200 import loss as LS
    g = torch.Generator().manual_seed(2)
    xs, xt = torch.randn(40, 33, generator=g), torch.randn(37, 33, generator=g) + 0.4
    ys, yt = torch.randn(40, 9, generator=g), torch.randn(37, 9, generator=g) - 0.1
    for name in ("mmd", "jan"):
        leaves = [t.to(_dev()).requires_grad_(True) for t in (xs, xt, ys, yt)]
        ref = [t.double().requires_grad_(True) for t in (xs, xt, ys, yt)]
        if name == "mmd":
            got = TF.mmd_loss(leaves[0], leaves[1], 2.0, 5)
            want = LS.mmd_rbf(ref[0][:37], ref[1][:37], 2.0, 5)
        else:
            got = TF.jan_loss([leaves[2], leaves[0]], [leaves[3], leaves[1]])
            want = LS.JAN([ref[2][:37], ref[0][:37]], [ref[3][:37], ref[1][:37]])
        (3.0 * got).backward()
        (3.0 * want).backward()
        assert_close(got.detach().cpu(), want.detach(), 1e-4, name)
        for a, b in zip(leaves, ref):
            if b.grad is not None:
                assert_close(a.grad.cpu(), b.grad, 1e-4, name + " grad")


@gpu
def test_autograd_wrappers_refuse_layers_of_unequal_rows():
    """The entry point reads Bs rows of every source layer and Bt of every target layer: layers of one domain with
    different row counts are refused before any launch, in either order."""
    from ta3n_b200 import Ta3nError
    from ta3n_b200 import functional as TF
    d = _dev()
    ys, xs = torch.randn(40, 9, device=d), torch.randn(38, 33, device=d)
    yt, xt = torch.randn(37, 9, device=d), torch.randn(37, 33, device=d)
    for src, tgt in (([ys, xs], [yt, xt]), ([xs[:36], ys[:37]], [xt, yt]), ([ys, xs[:37]], [yt, xt[:36]])):
        with pytest.raises(Ta3nError, match="one row count"):
            TF.jan_loss(src, tgt)
    with pytest.raises(Ta3nError, match="widths"):
        TF.mmd_loss(xs, yt)
    # equal counts per domain, Bs != Bt: gradients on every row, exactly 0 past the pairs
    leaves = [t.clone().requires_grad_(True) for t in (ys, torch.randn(40, 33, device=d), yt, xt)]
    TF.jan_loss(leaves[:2], leaves[2:]).backward()
    for t in leaves:
        assert t.grad.shape == t.shape and torch.isfinite(t.grad).all()
    assert not leaves[0].grad[37:].any() and not leaves[1].grad[37:].any()


# ---- GPU: TrainStep --------------------------------------------------------------------------------------------------
def _model(add_fc=1, T=5, C=7, fc_dim=256, drop=0.0, attn="TransAttn", attn_frame="none", ens="none", seed=3):
    from ta3n_b200.models import VideoModel
    torch.manual_seed(seed)
    m = VideoModel(C, "video", "trn-m", "RGB", train_segments=T, val_segments=T, add_fc=add_fc, fc_dim=fc_dim,
                   dropout_i=drop, dropout_v=drop, partial_bn=False, use_attn=attn, use_attn_frame=attn_frame,
                   ens_DA=ens, verbose=False)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for _, v in sorted(m.named_parameters()):
            if v.dim() > 1:
                v.add_(0.02 * torch.randn(v.shape, generator=g))
    return m.to(_dev()).train()


def _inputs(bs, bt, T, seed=9):
    from oracle import ta3n_oracle as orc
    g = torch.Generator().manual_seed(seed)
    xs = torch.randn(bs, T, orc.FEATURE_DIM, generator=g)
    xt = torch.randn(bt, T, orc.FEATURE_DIM, generator=g) * 1.2 - 0.3
    return xs, xt, torch.arange(bs) % 7


STEP_CASES = {
    # name: (dis, place, attn, attn_frame, add_fc, ens, mu, drop, (Bs, Bt), (ns, nt), alpha)
    "dan_attn": ("DAN", "YYN", "TransAttn", "none", 1, "none", 0.0, 0.0, (10, 7), (10, 7), 1.0),
    "dan_attn_drop": ("DAN", "YYN", "TransAttn", "none", 1, "none", 0.0, 0.5, (10, 7), (10, 7), 0.7),
    "jan_attn_drop": ("JAN", "YYN", "TransAttn", "none", 1, "none", 0.0, 0.5, (9, 12), (9, 12), 1.0),
    "dan_none_ynn": ("DAN", "YNN", "none", "none", 1, "none", 0.0, 0.0, (8, 8), (8, 8), 1.0),
    "jan_none": ("JAN", "YYN", "none", "none", 1, "none", 0.0, 0.5, (8, 6), (8, 6), 1.0),
    "dan_frame_attn": ("DAN", "NYN", "TransAttn", "TransAttn", 1, "none", 0.0, 0.5, (7, 9), (7, 9), 1.0),
    "dan_add_fc2": ("DAN", "YYNN", "TransAttn", "none", 2, "none", 0.0, 0.5, (10, 7), (10, 7), 1.0),
    "dan_mcd_mu07": ("DAN", "YYN", "TransAttn", "none", 1, "MCD", 0.7, 0.0, (8, 6), (8, 6), 1.0),
    "dan_mcd_mu07_drop": ("DAN", "YYN", "TransAttn", "none", 1, "MCD", 0.7, 0.5, (8, 6), (8, 6), 1.0),
    "jan_mcd_mu07_drop": ("JAN", "YYN", "TransAttn", "none", 1, "MCD", 0.7, 0.5, (8, 6), (8, 6), 0.5),
    "dan_short": ("DAN", "YYN", "TransAttn", "none", 1, "none", 0.0, 0.5, (10, 7), (6, 4), 1.0),
    "jan_short": ("JAN", "YYN", "TransAttn", "none", 1, "none", 0.0, 0.5, (10, 7), (3, 5), 1.0),
}


@pytest.fixture(params=["fp32", "tf32x3"])
def engine(request):
    import ta3n_b200
    ta3n_b200.set_gemm_engine(request.param)
    yield request.param
    ta3n_b200.set_gemm_engine("tf32x3")


@gpu
@pytest.mark.parametrize("case", list(STEP_CASES))
def test_train_step_matches_fp64_oracle(case, engine):
    """One TrainStep against the fp64 oracle: loss, loss_d and every gradient; with dropout on, the oracle takes the
    masks rebuilt from the counter RNG with the step's seeds (MCD: both passes' masks, which differ, so the term must
    read pass 1's target logits, not those pass 2 writes over them) and the ReLU pattern the step realised."""
    from oracle import add_fc_oracle as afo
    from oracle import mcd_oracle as mcd
    from oracle import ta3n_oracle as orc
    from ta3n_b200.train import TrainStep
    dis, place, attn, attn_frame, add_fc, ens, mu, drop, (Bs, Bt), (ns, nt), alpha = STEP_CASES[case]
    T = 5
    m = _model(add_fc, T=T, drop=drop, attn=attn, attn_frame=attn_frame, ens=ens)
    cfg = orc.PathConfig(num_class=7, num_segments=T, fc_dim=256, dropout_i=drop, dropout_v=drop, use_attn=attn,
                         use_attn_frame=attn_frame, ens_DA=ens)
    params = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    xs, xt, labels = _inputs(ns, nt, T)
    step = TrainStep(m, Bs, Bt, BETA, use_graph=False, dis_DA=dis, alpha=alpha, place_dis=tuple(place), mu=mu)
    loss = step(xs.pin_memory(), xt.pin_memory(), labels)
    torch.cuda.synchronize()
    masks = masks2 = gates2 = None
    key = int(step.step_counter.item())
    if drop > 0:
        masks = afo.train_step_masks(key, Bs, Bt, T, cfg.shared_dim, cfg.video_dim, drop, drop, add_fc, ns=ns, nt=nt)
        if ens == "MCD":
            masks2 = mcd.train_step_pass2_masks(key, Bt, T, cfg.shared_dim, cfg.video_dim, drop, drop, nt=nt)
    p64 = {k: v.double() if v.dtype.is_floating_point else v for k, v in params.items()}
    gates = afo.activation_pattern(p64, xs.double(), xt.double(), BETA, cfg, add_fc, masks)
    if add_fc == 1:
        # the ReLU pattern the step realised (a unit near 0 may flip under tf32x3), flip-bounded as elsewhere
        from tests.test_gpu_parity import FLIP_BOUND
        from tests.pinned_pattern import realised_gates
        ones = lambda r: torch.ones(r, cfg.shared_dim, dtype=torch.bool)              # noqa: E731
        kept = ones((ns + nt) * T) if masks is None else torch.cat([masks["i_source"], masks["i_target"]]).bool()
        frames = lambda t: torch.cat([t[:ns * T], t[Bs * T:Bs * T + nt * T]]).cpu()    # noqa: E731
        videos = lambda t: torch.cat([t[:ns], t[Bs:Bs + nt]]).cpu()                    # noqa: E731
        gates, flips, total = realised_gates(step.bufs.pool, frames, videos, kept, gates, True, True)
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
    kw = dict(place_dis=place, add_fc=add_fc, train=drop > 0, masks=masks, gates=gates, mu=mu, masks2=masks2,
              gates2=gates2)
    l64, d64, g64 = dor.dis_train_step(p64, xs.double(), xt.double(), labels, BETA, cfg, dis, alpha, **kw)
    _, d32, g32 = dor.dis_train_step(params, xs, xt, labels, BETA, cfg, dis, alpha, **kw)
    assert_close(loss.cpu()[0], l64, 2e-4, "loss")
    assert_close(step.loss_d.cpu()[0], d64, 2e-4, "loss_d", noise=abs(d32.double() - d64).item() * 8)
    named = dict(m.named_parameters())
    scale = {"fp32": 1.0, "tf32x3": 8.0}[engine]
    for name, g in g64.items():
        if g is None:
            continue
        noise = (g32[name].double() - g).norm().item() * scale
        assert_close(named[name].grad, g, {"fp32": 4e-4, "tf32x3": 1e-3}[engine], f"grad {name}", noise=noise)


@gpu
@pytest.mark.parametrize("dis", ["DAN", "JAN"])
def test_batch_without_target_rows_adds_nothing(dis):
    """A batch with no real target row: the step equals the plain step bit for bit, and loss_d is 0."""
    from ta3n_b200.train import TrainStep
    xs, xt, labels = _inputs(6, 4, 5)
    m_a = _model()
    m_b = copy.deepcopy(m_a)
    plain = TrainStep(m_a, 6, 4, BETA, seed=3)
    step = TrainStep(m_b, 6, 4, BETA, seed=3, dis_DA=dis, alpha=1.0)
    la, lb = plain(xs, xt[:0], labels).clone(), step(xs, xt[:0], labels).clone()
    torch.cuda.synchronize()
    assert torch.equal(la, lb) and step.loss_d.item() == 0.0
    assert torch.equal(plain.flat_grad, step.flat_grad)


@gpu
@pytest.mark.parametrize("dis", ["DAN", "JAN"])
def test_eager_graph_and_set_alpha(dis):
    """Eager == graph bit for bit over three SGD steps (dropout on, a short batch among them); then, with no
    optimizer, set_alpha between replays changes the loss by (alpha' - alpha) * loss_d without a re-capture."""
    from ta3n_b200.train import SGDNesterov, TrainStep
    xs, xt, labels = _inputs(8, 6, 5)
    runs = []
    for use_graph in (False, True):
        m = _model(drop=0.5)
        step = TrainStep(m, 8, 6, BETA, use_graph=use_graph, optimizer=SGDNesterov(lr=0.01), seed=11, dis_DA=dis,
                         alpha=0.5)
        if use_graph:
            step.step_counter.fill_(0)       # the capture's warm-up advanced the dropout counter
        losses = []
        for i in range(3):
            n = (8, 6) if i != 1 else (5, 3)
            losses.append(step(xs[:n[0]], xt[:n[1]], labels[:n[0]]).clone())
        torch.cuda.synchronize()
        runs.append((torch.cat(losses), step.flat_param.clone()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    step = TrainStep(_model(), 8, 6, BETA, dis_DA=dis, alpha=0.25)
    n_capture = step.graphs[0][0]
    l1, d1 = step(xs, xt, labels).item(), step.loss_d.item()
    with pytest.raises(ValueError, match="alpha_dann"):
        step.set_alpha(-0.5)
    step.set_alpha(1.25)
    l2, d2 = step(xs, xt, labels).item(), step.loss_d.item()
    assert step.graphs[0][0] is n_capture and d1 == d2 and d1 > 0
    assert l2 - l1 == pytest.approx(1.0 * d1, rel=1e-4, abs=1e-6)


def _stock_loop(m, xs, xt, labels, opt_name, n, dis, alpha):
    from ta3n_b200 import loss as LS
    params = list(m.parameters())
    opt = torch.optim.SGD(params, 0.01, momentum=0.9, weight_decay=1e-4, nesterov=True) if opt_name == "sgd" else \
        torch.optim.Adam(params, 1e-3, weight_decay=1e-4)
    d = _dev()
    for _ in range(n):
        opt.zero_grad(set_to_none=True)
        outs = m(xs.to(d), xt.to(d), list(BETA), 0, is_train=True, reverse=False)
        loss = LS.ta3n_loss(outs, labels.to(d), 0.003) + alpha * LS.discrepancy_loss(outs[4], outs[9], dis)
        loss.backward()
        torch.nn.utils.clip_grad_norm_([p for p in params if p.grad is not None], 20.0)
        opt.step()


@gpu
@pytest.mark.parametrize("opt_name", ["sgd", "adam"])
@pytest.mark.parametrize("dis", ["DAN", "JAN"])
def test_three_steps_match_the_stock_autograd_loop(opt_name, dis):
    from ta3n_b200.train import Adam, SGDNesterov, TrainStep
    xs, xt, labels = _inputs(8, 6, 5)
    m_a = _model()
    m_b = copy.deepcopy(m_a)
    opt = SGDNesterov(lr=0.01) if opt_name == "sgd" else Adam(lr=1e-3)
    step = TrainStep(m_a, 8, 6, BETA, optimizer=opt, dis_DA=dis, alpha=2.0)
    for _ in range(3):
        step(xs, xt, labels)
    torch.cuda.synchronize()
    _stock_loop(m_b, xs, xt, labels, opt_name, 3, dis, 2.0)
    pb = dict(m_b.named_parameters())
    for name, p in m_a.named_parameters():
        assert_close(p.detach(), pb[name].detach(), 1e-4, name)


@gpu
def test_resume_from_state_dict_is_bit_identical():
    from ta3n_b200.train import Adam, TrainStep
    xs, xt, labels = _inputs(6, 5, 5)
    m_a = _model(drop=0.5)
    m_b = copy.deepcopy(m_a)
    kw = dict(optimizer=Adam(lr=1e-3), seed=5, dis_DA="DAN", alpha=0.8)
    a = TrainStep(m_a, 6, 5, BETA, **kw)
    for _ in range(4):
        a(xs, xt, labels)
    b0 = TrainStep(m_b, 6, 5, BETA, **kw)
    for _ in range(2):
        b0(xs, xt, labels)
    sd = copy.deepcopy(b0.state_dict())
    params = copy.deepcopy(m_b.state_dict())
    m_c = _model(drop=0.5, seed=99)
    m_c.load_state_dict(params)
    c = TrainStep(m_c, 6, 5, BETA, **kw)
    c.load_state_dict(sd)
    for _ in range(2):
        c(xs, xt, labels)
    torch.cuda.synchronize()
    assert torch.equal(a.flat_param, c.flat_param)


@gpu
def test_meters_equal_the_reference_average_meters():
    """Over an epoch with a short last batch, stats() / stats_async(): losses_d is updated with the unscaled term and
    the real source rows (main.py:504), the loss meter with the loss the step reports, which includes alpha * loss_d
    (main.py:569: losses.update(loss.item()), n = 1)."""
    from oracle.train_stats_oracle import AverageMeter
    from ta3n_b200.train import TrainStep
    xs, xt, labels = _inputs(8, 6, 5)
    step = TrainStep(_model(drop=0.5), 8, 6, BETA, dis_DA="JAN", alpha=0.6, stats=True)
    ref_d, ref_l = AverageMeter(), AverageMeter()
    for n in ((8, 6), (8, 6), (5, 2)):
        loss = step(xs[:n[0]], xt[:n[1]], labels[:n[0]]).item()
        ref_d.update(step.loss_d.item(), n[0])
        ref_l.update(loss)
    st, snap = step.stats(), step.stats_async().result()
    for got in (st, snap):
        assert got.loss_d.count == ref_d.count == 21
        assert got.loss_d.val == ref_d.val and got.loss_d.sum == pytest.approx(ref_d.sum, rel=1e-12)
        assert got.loss_d.avg == pytest.approx(ref_d.avg, rel=1e-12)
        assert got.loss.avg == pytest.approx(ref_l.avg, rel=1e-6)
    step.reset_stats()
    assert step.stats().loss_d.count == 0


# launches per step of the plain legacy step at this file's shape (T=5, fc_dim 256, 8 + 6 videos, tf32x3), as the
# parent of the discrepancy change counted them: 34 without an optimizer, 36 with SGD and clipping
PLAIN_LAUNCHES = {False: 34, True: 36}


@gpu
@pytest.mark.parametrize("with_opt", [False, True])
@pytest.mark.parametrize("dis", ["none", "DAN", "JAN"])
def test_launches_the_term_adds(dis, with_opt):
    """dis_DA='none' issues the plain step's launches, unchanged; the term adds three."""
    import ta3n_b200
    from ta3n_b200.train import SGDNesterov, TrainStep
    ta3n_b200.set_gemm_engine("tf32x3")
    m = _model()
    step = TrainStep(m, 8, 6, BETA, dis_DA=dis, optimizer=SGDNesterov(lr=0.01) if with_opt else None)
    assert step.launches_per_step == PLAIN_LAUNCHES[with_opt] + (0 if dis == "none" else 3)
