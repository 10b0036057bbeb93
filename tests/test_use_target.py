"""TrainStep(use_target='Sv' | 'none'): supervised target labels in the class loss, and the source-only baseline.

CPU: the options TrainStep refuses with either value, the autograd loss (``loss.ta3n_loss(use_target=...)``) against
main.py:442-446's composition, and the argument checks of the three new C entries.
GPU: the Sv loss entry and the Sv meters entry against fp64 restatements, also at cfg5's 1024 rows (the meters' 128
CTA partials); the labelled gather against the plain one;
TrainStep iterations against the stock autograd loop with torch.optim (fp32 engine); bit-identical eager / graph /
reruns / resume, device sampler and double buffering; 'uSv' equal to the default; the launches of 'none' and the
parameters it leaves alone; the meters.
"""
import copy
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import ta3n_oracle as orc
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


@pytest.mark.parametrize("use_target", ["Sv", "none"])
def test_train_step_refusals(use_target, monkeypatch):
    from ta3n_b200 import Ta3nError, train
    from ta3n_b200.train import SGDNesterov, TrainStep
    m = _cpu_model()
    kw = dict(use_target=use_target, optimizer=SGDNesterov(lr=0.01))
    with pytest.raises(NotImplementedError, match="legacy"):
        TrainStep(m, 4, 4, beta=BETA, mode="phased", **kw)
    with pytest.raises(NotImplementedError, match="step program"):
        TrainStep(m, 4, 4, beta=BETA, class_weight=torch.ones(5), **kw)
    with pytest.raises(NotImplementedError, match="step program"):
        TrainStep(m, 4, 4, beta=BETA, domain_weight=(1.0, 0.5), **kw)
    with pytest.raises(NotImplementedError, match="step program"):
        TrainStep(m, 4, 4, beta=[-1.0, 0.75, 0.5], **kw)
    mcd = _cpu_model(ens_DA="MCD")
    with pytest.raises(NotImplementedError if use_target == "Sv" else ValueError, match="MCD"):
        TrainStep(mcd, 4, 4, beta=BETA, **kw)
    # the accepted configuration passes every check and stops at the device; under 'none' the DA options are ignored
    with pytest.raises(Ta3nError, match="CUDA"):
        TrainStep(m, 4, 4, beta=BETA, **kw)
    if use_target == "none":
        with pytest.raises(Ta3nError, match="CUDA"):
            TrainStep(m, 4, 4, beta=BETA, dis_DA="CORAL", alpha=-1.0, add_loss_DA="bogus", **kw)
    monkeypatch.setattr(train.dist, "is_initialized", lambda: True)
    monkeypatch.setattr(train.dist, "get_world_size", lambda group=None: 2)
    monkeypatch.setattr(train.dist, "get_rank", lambda group=None: 0)
    with pytest.raises(NotImplementedError, match="single rank"):
        TrainStep(m, 4, 4, beta=BETA, **kw)


def test_unknown_use_target_and_default():
    from ta3n_b200 import Ta3nError
    from ta3n_b200.train import TrainStep
    m = _cpu_model()
    for bad in ("uSv ", "sv", "None", None):
        with pytest.raises(ValueError, match="use_target"):
            TrainStep(m, 4, 4, beta=BETA, use_target=bad)
    with pytest.raises(Ta3nError, match="CUDA"):
        TrainStep(m, 4, 4, beta=BETA, use_target="uSv")


def _outputs(Bs, Bt, C=6, R=4, seed=0):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64, requires_grad=True)      # noqa: E731
    out_s, out_t = r(Bs, C), r(Bt, C)
    pd_s, pd_t = [r(Bs, R, 2), r(Bs, 2), r(Bs * 5, 2)], [r(Bt, R, 2), r(Bt, 2), r(Bt * 5, 2)]
    return (None, out_s, None, pd_s, None, None, out_t, None, pd_t, None), torch.arange(Bs) % C, \
        (torch.arange(Bt) * 5 + 1) % C


@pytest.mark.parametrize("Bs,Bt", [(6, 4), (5, 0)])
def test_autograd_loss_with_use_target(Bs, Bt):
    """loss.ta3n_loss: 'Sv' = CE over cat(out_s, out_t) / cat(labels) (main.py:442-446) + the unsupervised terms;
    'none' = CE(out_s) alone; 'uSv' = the default."""
    from ta3n_b200 import loss as LS
    outs, ls, lt = _outputs(Bs, Bt)
    out_s, out_t = outs[1], outs[6]
    base = LS.ta3n_loss(outs, ls, 0.3)
    assert torch.equal(LS.ta3n_loss(outs, ls, 0.3, use_target="uSv"), base)
    sv = LS.ta3n_loss(outs, ls, 0.3, use_target="Sv", label_target=lt)
    da = base - F.cross_entropy(out_s, ls)
    want = F.cross_entropy(torch.cat([out_s, out_t]), torch.cat([ls, lt])) + da
    assert sv.item() == pytest.approx(want.item(), rel=1e-12)
    assert torch.equal(LS.ta3n_loss(outs, ls, 0.3, use_target="none"), F.cross_entropy(out_s, ls))
    with pytest.raises(ValueError, match="label_target"):
        LS.ta3n_loss(outs, ls, 0.3, use_target="Sv")
    with pytest.raises(ValueError, match="label_target"):
        LS.ta3n_loss(outs, ls, 0.3, use_target="Sv", label_target=torch.zeros(Bt + 1, dtype=torch.long))
    with pytest.raises(ValueError, match="use_target"):
        LS.ta3n_loss(outs, ls, 0.3, use_target="semi")


@pytest.fixture(scope="module")
def lib():
    from ta3n_b200 import _lib
    return _lib.load()


def test_sv_loss_entry_validates_arguments_without_gpu(lib):
    def call(**kw):
        a = dict(pv=16, lab=32, lt=48, rel=64, dom=80, frame=96, Bs=4, Bt=4, T=5, R=4, C=12, ws=4096, ws_bytes=1 << 12)
        a.update(kw)
        return lib.ta3n_loss_fwd_bwd_sv(a["pv"], a["lab"], a["lt"], a["rel"], a["dom"], a["frame"], a["Bs"], a["Bt"],
                                        a["T"], a["R"], a["C"], 0.003, 15, None, 112, 128, 144, 160, 176, a["ws"],
                                        a["ws_bytes"], None)
    assert call(lt=None) == 1 and b"ta3n_loss_fwd_bwd_sv" in lib.ta3n_last_error() and \
        b"target labels" in lib.ta3n_last_error()
    assert call(Bs=0) == 1 and b"bad sizes" in lib.ta3n_last_error()
    assert call(C=0) == 1
    assert call(pv=None) == 1 and b"null input" in lib.ta3n_last_error()
    assert call(ws_bytes=16) == 2 and b"ta3n_loss_fwd_bwd_sv: workspace too small" in lib.ta3n_last_error()


def test_sv_meters_entry_validates_arguments_without_gpu(lib):
    k2 = (C.c_int * 2)(1, 5)
    dw = (C.c_float * 2)(1.0, 1.0)

    def call(**kw):
        a = dict(pv=16, lab=32, lt=48, rel=64, dom=80, frame=96, loss=112, Bs=4, Bt=4, flags=15, k=k2, n_k=2,
                 acc=4096, prec=8192, ws=16384, ws_bytes=1 << 12)
        a.update(kw)
        return lib.ta3n_train_stats_accumulate_sv(a["pv"], a["lab"], a["lt"], a["rel"], a["dom"], a["frame"],
                                                  a["loss"], a["Bs"], a["Bt"], 5, 4, 12, a["flags"], None, None, dw,
                                                  a["n_k"], a["k"], a["acc"], a["prec"], a["ws"], a["ws_bytes"], None)
    for kw, msg in ((dict(lt=None), b"null target labels"), (dict(prec=None), b"prec_sum"),
                    (dict(prec=8196), b"8-byte aligned"), (dict(acc=None), b"null accumulator"),
                    (dict(acc=4100), b"8-byte aligned"), (dict(Bs=0), b"bad sizes"), (dict(flags=16), b"flags"),
                    (dict(k=(C.c_int * 2)(1, 13)), b"outside [1, C=12]"), (dict(pv=None), b"null input"),
                    (dict(ws_bytes=16), b"workspace too small")):
        rc = call(**kw)
        err = lib.ta3n_last_error()
        assert rc in (1, 2) and b"ta3n_train_stats_accumulate_sv" in err and msg in err, (kw, err)


def test_labelled_gather_validates_arguments_without_gpu(lib):
    ok = dict(bank_s=256, n_rows_s=10, rows_s=512, labels_s=768, n_epoch_s=10, batch_s=4, x_s=1024, y_s=1280,
              bank_t=1536, n_rows_t=8, rows_t=1792, labels_t=3072, n_epoch_t=8, batch_t=3, x_t=2048, y_t=3328,
              row_floats=40, valid=2304, state=2560, stream=None)

    def call(**kw):
        a = dict(ok)
        a.update(kw)
        return lib.ta3n_gather_batch_labelled(*a.values())
    for kw, msg in ((dict(labels_t=None), b"null target label list"), (dict(y_t=None), b"null target label list"),
                    (dict(x_t=None), b"null target"), (dict(batch_t=0), b"batch sizes"),
                    (dict(row_floats=42), b"multiple of 4"), (dict(x_s=1028), b"16-byte aligned")):
        assert call(**kw) == 1, kw
        err = lib.ta3n_last_error()
        assert b"ta3n_gather_batch_labelled" in err and msg in err, (kw, err)


# ------------------------------------------------------------------------------------------------
# GPU: the entries alone
# ------------------------------------------------------------------------------------------------
def _dev():
    return torch.device("cuda:0")


def _P(t):
    return None if t is None else t.data_ptr()


def _loss_inputs(Bs, Bt, T, R, C, seed=1):
    g = torch.Generator().manual_seed(seed)
    M = Bs + Bt
    pv = torch.randn(M, C, generator=g) * 3
    rel, dom, frame = torch.randn(M, R, 2, generator=g), torch.randn(M, 2, generator=g), \
        torch.randn(M * T, 2, generator=g)
    ls = torch.randint(0, C, (Bs,), generator=g)
    lt = torch.randint(0, C, (Bt,), generator=g)
    return pv, rel, dom, frame, ls, lt


def _loss_call(lib, entry, pv, rel, dom, frame, ls, lt, Bs, Bt, T, R, C, flags, gamma, valid):
    d = _dev()
    M = Bs + Bt
    ins = [t.to(d).contiguous() for t in (pv, rel, dom, frame, ls)]
    lt_d = lt.to(d).contiguous() if lt is not None else None
    loss = torch.zeros(1, device=d)
    g = [torch.full(s, float("nan"), device=d) for s in ((M, C), (M, R, 2), (M, 2), (M * T, 2))]
    ws = torch.zeros(lib.ta3n_loss_workspace_bytes(M) // 4 + 64, device=d)
    v = torch.tensor(valid, device=d, dtype=torch.int32)
    args = [_P(ins[0]), _P(ins[4])] + ([_P(lt_d)] if entry == "sv" else []) + \
        [_P(ins[1]), _P(ins[2]), _P(ins[3]), Bs, Bt, T, R, C, gamma, flags, _P(v), _P(loss)] + [_P(x) for x in g] + \
        [_P(ws), ws.numel() * 4, None]
    fn = lib.ta3n_loss_fwd_bwd_sv if entry == "sv" else lib.ta3n_loss_fwd_bwd
    from ta3n_b200._lib import check
    check(fn(*args))
    torch.cuda.synchronize()
    return loss.cpu(), [x.cpu() for x in g]


def _loss_fp64(pv, rel, dom, frame, ls, lt, Bs, vs, vt, T, R, flags, gamma):
    """main.py:442-446, 508-538, 559-562 under Sv on the real rows, in fp64, with autograd gradients."""
    leaves = [t.double().clone().requires_grad_(True) for t in (pv, rel, dom, frame)]
    pv_, rel_, dom_, frame_ = leaves
    real = torch.cat([torch.arange(vs), Bs + torch.arange(vt)])
    z = pv_[real]
    loss = F.cross_entropy(z, torch.cat([ls[:vs], lt[:vt]]))
    d = torch.cat([torch.zeros(vs, dtype=torch.long), torch.ones(vt, dtype=torch.long)])
    if flags & 1:
        loss = loss + F.cross_entropy(rel_[real].reshape(-1, 2), d.repeat_interleave(R))
    if flags & 2:
        loss = loss + F.cross_entropy(dom_[real], d)
    if flags & 4:
        fr = frame_.view(-1, T, 2)[real].reshape(-1, 2)
        loss = loss + F.cross_entropy(fr, d.repeat_interleave(T))
    if flags & 8:
        from ta3n_b200.loss import attentive_entropy
        loss = loss + gamma * attentive_entropy(z, dom_[real])
    grads = torch.autograd.grad(loss, leaves)
    return loss.detach(), grads


@gpu
@pytest.mark.parametrize("C", [5, 97, 1000])
@pytest.mark.parametrize("valid", [(9, 7), (6, 3), (9, 0), (1, 7)])
def test_sv_loss_entry_matches_fp64(C, valid):
    """The Sv loss heads against the fp64 restatement at fp32 grade, loss and every gradient, padded rows zero."""
    from ta3n_b200 import _lib
    lib = _lib.load()
    Bs, Bt, T, R = 9, 7, 5, 4
    vs, vt = valid
    pv, rel, dom, frame, ls, lt = _loss_inputs(Bs, Bt, T, R, C)
    loss, g = _loss_call(lib, "sv", pv, rel, dom, frame, ls, lt, Bs, Bt, T, R, C, 15, 0.3, valid)
    want, wg = _loss_fp64(pv, rel, dom, frame, ls, lt, Bs, vs, vt, T, R, 15, 0.3)
    assert abs(loss.double().item() - want.item()) <= 2e-6 * abs(want.item()) + 1e-6
    pad = torch.ones(Bs + Bt, dtype=torch.bool)
    pad[:vs] = False
    pad[Bs:Bs + vt] = False
    for got, ref, name in zip(g, wg, ("pred_video", "pred_rel", "pred_dom", "pred_frame")):
        rows = got.view(Bs + Bt, -1)
        assert torch.all(rows[pad] == 0), name
        real = ref.view(Bs + Bt, -1)[~pad]
        assert_close(rows[~pad], real, 2e-5, name, noise=1e-9)


@gpu
@pytest.mark.parametrize("C", [30, 1000])
@pytest.mark.parametrize("valid", [(512, 512), (500, 311)])
def test_sv_loss_entry_at_full_size(C, valid):
    """The Sv loss entry at cfg5's M = 1024 rows (Bs = Bt = 512), where its grid-stride loops make several trips:
    the loss and every gradient against fp64, per row of the class logits' gradient too, padded rows zero."""
    from ta3n_b200 import _lib
    lib = _lib.load()
    Bs, Bt, T, R = 512, 512, 5, 4
    vs, vt = valid
    pv, rel, dom, frame, ls, lt = _loss_inputs(Bs, Bt, T, R, C, seed=C)
    loss, g = _loss_call(lib, "sv", pv, rel, dom, frame, ls, lt, Bs, Bt, T, R, C, 15, 0.3, valid)
    want, wg = _loss_fp64(pv, rel, dom, frame, ls, lt, Bs, vs, vt, T, R, 15, 0.3)
    assert abs(loss.double().item() - want.item()) <= 2e-6 * abs(want.item()) + 1e-6
    pad = torch.ones(Bs + Bt, dtype=torch.bool)
    pad[:vs] = False
    pad[Bs:Bs + vt] = False
    for got, ref, name in zip(g, wg, ("pred_video", "pred_rel", "pred_dom", "pred_frame")):
        rows = got.view(Bs + Bt, -1)
        assert torch.all(rows[pad] == 0), name
        real, got_real = ref.view(Bs + Bt, -1)[~pad], rows[~pad].double()
        assert_close(got_real, real, 2e-5, name, noise=1e-9)
        err, den = (got_real - real).norm(dim=1), real.norm(dim=1)
        bad = err > 2e-5 * den + 1e-9
        assert not bool(bad.any()), f"{name}: row {int(torch.nonzero(bad)[0, 0])} off"


@gpu
def test_sv_loss_entry_equals_the_plain_entry_without_target_rows_and_handles_nan():
    """With no real target row the Sv entry is the plain entry, bit for bit; a NaN target logit makes the loss NaN and
    leaves the other rows' gradients finite."""
    from ta3n_b200 import _lib
    lib = _lib.load()
    Bs, Bt, T, R, C = 9, 7, 5, 4, 11
    pv, rel, dom, frame, ls, lt = _loss_inputs(Bs, Bt, T, R, C, seed=4)
    for flags in (0, 7, 15):
        a = _loss_call(lib, "sv", pv, rel, dom, frame, ls, lt, Bs, Bt, T, R, C, flags, 0.3, (6, 0))
        b = _loss_call(lib, "plain", pv, rel, dom, frame, ls, None, Bs, Bt, T, R, C, flags, 0.3, (6, 0))
        assert torch.equal(a[0], b[0]) and all(torch.equal(x, y) for x, y in zip(a[1], b[1])), flags
    pv[Bs + 2, 3] = float("nan")
    loss, g = _loss_call(lib, "sv", pv, rel, dom, frame, ls, lt, Bs, Bt, T, R, C, 0, 0.3, (Bs, Bt))
    assert torch.isnan(loss).all() and torch.isfinite(g[0][:Bs]).all()


def _stats_call(lib, acc, prec, ws, pv, rel, dom, frame, ls, lt, loss, Bs, Bt, T, R, n_cls, flags, valid, k):
    from ta3n_b200._lib import check
    v = torch.tensor(valid, device=_dev(), dtype=torch.int32)
    dw = (C.c_float * 2)(1.0, 1.0)
    kk = (C.c_int * len(k))(*k)
    check(lib.ta3n_train_stats_accumulate_sv(
        _P(pv), _P(ls), _P(lt), _P(rel), _P(dom), _P(frame), _P(loss), Bs, Bt, T, R, n_cls, flags, _P(v), None, dw,
        len(k), kk, _P(acc), _P(prec), _P(ws), ws.numel(), None))


@gpu
def test_sv_meters_entry_over_an_epoch():
    """An epoch with a short last batch: loss_c and top-1 / top-5 are the AverageMeter folds of main.py:446-450 and
    :565-571 under Sv (values over source and target rows, n = the real source rows); replays are bit-identical."""
    from oracle.train_stats_oracle import AverageMeter
    from ta3n_b200 import _lib
    from ta3n_b200.train import _STATS_WORDS, parse_train_stats, sv_prec
    lib = _lib.load()
    d = _dev()
    Bs, Bt, T, R, C = 12, 10, 5, 4, 9
    batches = [(12, 10), (12, 10), (7, 3), (5, 0)]
    ws = torch.zeros(lib.ta3n_train_stats_workspace_bytes(Bs + Bt), device=d, dtype=torch.uint8)
    runs = []
    for _ in range(2):
        acc = torch.zeros(_STATS_WORDS, device=d, dtype=torch.int64)
        prec = torch.zeros(4, device=d, dtype=torch.float64)
        mc, m1, m5 = AverageMeter(), AverageMeter(), AverageMeter()
        for i, (vs, vt) in enumerate(batches):
            pv, rel, dom, frame, ls, lt = _loss_inputs(Bs, Bt, T, R, C, seed=20 + i)
            ins = [t.to(d).contiguous() for t in (pv, rel, dom, frame, ls, lt)]
            loss = torch.tensor([1.5 + i], device=d)
            _stats_call(lib, acc, prec, ws, *ins, loss, Bs, Bt, T, R, C, 15, (vs, vt), (1, 5))
            z = torch.cat([pv[:vs], pv[Bs:Bs + vt]]).double()
            y = torch.cat([ls[:vs], lt[:vt]])
            mc.update(F.cross_entropy(z, y).item(), vs)
            rank = (z > z.gather(1, y[:, None])).sum(1)
            m1.update(100.0 * (rank < 1).sum().item() / (vs + vt), vs)
            m5.update(100.0 * (rank < 5).sum().item() / (vs + vt), vs)
        torch.cuda.synchronize()
        st = parse_train_stats(acc.cpu().numpy(), (1, 5))
        sv_prec(st, prec.cpu().numpy())
        assert st.loss_c.count == mc.count == 36 and st.loss_c.avg == pytest.approx(mc.avg, rel=1e-6)
        assert st.top1.count == 36 and st.top1.avg == pytest.approx(m1.avg, rel=1e-12)
        assert st.top5.avg == pytest.approx(m5.avg, rel=1e-12)
        assert st.top1.val == pytest.approx(m1.val, rel=1e-12)
        runs.append((acc.cpu(), prec.cpu()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


@gpu
@pytest.mark.parametrize("C", [5, 30, 101])
def test_sv_meters_entry_at_full_size(C):
    """The Sv meters at M = 1024 rows: 128 CTAs whose partials the last one to arrive folds.  An epoch of four
    batches with a short last one against the oracle's fold (use_target_oracle.fold, train_stats_oracle.label_rank's
    tie rule), and a second run of the epoch bit-identical to the first."""
    from oracle import train_stats_oracle as tso
    from oracle import use_target_oracle as uto
    from ta3n_b200 import _lib
    from ta3n_b200.train import _STATS_WORDS, parse_train_stats, sv_prec
    lib = _lib.load()
    d = _dev()
    Bs, Bt, T, R = 512, 512, 5, 4
    batches = [(512, 512), (512, 512), (512, 512), (300, 211)]
    ws = torch.zeros(lib.ta3n_train_stats_workspace_bytes(Bs + Bt), device=d, dtype=torch.uint8)
    runs = []
    for _ in range(2):
        acc = torch.zeros(_STATS_WORDS, device=d, dtype=torch.int64)
        prec = torch.zeros(4, device=d, dtype=torch.float64)
        steps = []
        for i, (vs, vt) in enumerate(batches):
            pv, rel, dom, frame, ls, lt = _loss_inputs(Bs, Bt, T, R, C, seed=40 + i)
            ins = [t.to(d).contiguous() for t in (pv, rel, dom, frame, ls, lt)]
            loss = torch.tensor([1.5 + i], device=d)
            _stats_call(lib, acc, prec, ws, *ins, loss, Bs, Bt, T, R, C, 15, (vs, vt), (1, 5))
            z = torch.cat([pv[:vs], pv[Bs:Bs + vt]]).double().numpy()
            y = torch.cat([ls[:vs], lt[:vt]]).numpy()
            rank = tso.label_rank(z, y)
            steps.append({"loss": None, "loss_c": (float(tso._weighted_ce(z, y, None, np.float64)), vs),
                          "loss_a": None, "loss_e": None, "loss_s": None,
                          "correct": (int((rank < 1).sum()), int((rank < 5).sum())), "rows": vs + vt, "n": vs})
        torch.cuda.synchronize()
        want = uto.fold(steps)
        st = parse_train_stats(acc.cpu().numpy(), (1, 5))
        sv_prec(st, prec.cpu().numpy())
        assert st.loss_c.count == want["loss_c"].count == 1836
        assert st.loss_c.avg == pytest.approx(want["loss_c"].avg, rel=1e-6)
        assert st.loss_c.val == pytest.approx(want["loss_c"].val, rel=1e-6)
        for k in ("top1", "top5"):
            got = getattr(st, k)
            assert got.count == want[k].count and got.avg == pytest.approx(want[k].avg, rel=1e-12), k
            assert got.val == pytest.approx(want[k].val, rel=1e-12), k
        if C == 5:
            assert st.top5.avg == 100.0
        runs.append((acc.cpu(), prec.cpu()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


@gpu
def test_labelled_gather_equals_the_plain_gather(tmp_path):
    """ta3n_gather_batch_labelled fills what ta3n_gather_batch fills, bit for bit, plus the target labels of the
    loader's batch (0 on padded rows), over a whole epoch with a short last batch."""
    from ta3n_b200 import dataset as D
    from tests.test_device_sampler import _banks
    T, F_, batch = 5, 64, (8, 5)
    sets, banks = _banks(tmp_path, T, F_, (21, None), (13, None), batch)
    a = D.DevicePairedSampler(banks[0], banks[1], batch, seed=3)
    b = D.DevicePairedSampler(banks[0], banks[1], batch, seed=3)
    b.enable_target_labels()
    loader = D.PairedFeatureLoader(sets[0], sets[1], batch, seed=3, pin_memory=False)
    d = banks[0].device
    slot = lambda: (torch.full((batch[0], T, F_), 7.0, device=d), torch.full((batch[1], T, F_), 7.0, device=d),  # noqa
                    torch.full((batch[0],), -3, device=d, dtype=torch.int64), torch.zeros(2, device=d, dtype=torch.int32))
    assert a.start_epoch() == b.start_epoch() == len(loader)
    st = torch.cuda.current_stream().cuda_stream
    for (xs, ys), (xt, yt) in loader:
        sa, sb = slot(), slot()
        lt = torch.full((batch[1],), -3, device=d, dtype=torch.int64)
        a.enqueue_gather(*sa, st)
        b.enqueue_gather(*sb, st, labels_t=lt)
        torch.cuda.synchronize()
        for x, y in zip(sa, sb):
            assert torch.equal(x, y)
        nt = xt.shape[0]
        assert torch.equal(lt[:nt].cpu(), yt.long()) and torch.all(lt[nt:] == 0)
    assert torch.equal(a.state, b.state)


# ------------------------------------------------------------------------------------------------
# GPU: TrainStep
# ------------------------------------------------------------------------------------------------
def _model(T=5, C=7, drop=0.0, attn="TransAttn", attn_frame="none", add_fc=1, seed=3):
    from ta3n_b200.models import VideoModel
    torch.manual_seed(seed)
    m = VideoModel(C, "video", "trn-m", "RGB", train_segments=T, val_segments=T, fc_dim=256, dropout_i=drop,
                   dropout_v=drop, partial_bn=False, use_attn=attn, use_attn_frame=attn_frame, add_fc=add_fc,
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
    return xs, xt, torch.arange(bs) % 7, (torch.arange(bt) * 3 + 2) % 7


CASES = {
    # name: (use_target, attn, attn_frame, add_fc, T, (Bs, Bt), (ns, nt), add_loss_DA, pretrain, opt)
    "sv_attn": ("Sv", "TransAttn", "none", 1, 5, (8, 6), (8, 6), "attentive_entropy", False, "sgd"),
    "sv_noattn": ("Sv", "none", "none", 1, 5, (8, 6), (8, 6), "attentive_entropy", False, "sgd"),
    "sv_frame_t7": ("Sv", "TransAttn", "TransAttn", 1, 7, (7, 9), (7, 9), "attentive_entropy", False, "sgd"),
    "sv_add_fc2": ("Sv", "TransAttn", "none", 2, 5, (8, 6), (8, 6), "attentive_entropy", False, "sgd"),
    "sv_entropy": ("Sv", "TransAttn", "none", 1, 5, (8, 6), (8, 6), "target_entropy", False, "sgd"),
    "sv_pretrain": ("Sv", "TransAttn", "none", 1, 5, (8, 6), (8, 6), "attentive_entropy", True, "sgd"),
    "sv_short": ("Sv", "TransAttn", "none", 1, 5, (10, 7), (6, 3), "attentive_entropy", False, "sgd"),
    "sv_no_target": ("Sv", "TransAttn", "none", 1, 5, (8, 6), (5, 0), "attentive_entropy", False, "sgd"),
    "sv_adam": ("Sv", "TransAttn", "none", 1, 5, (8, 6), (8, 6), "attentive_entropy", False, "adam"),
    "none_attn": ("none", "TransAttn", "none", 1, 5, (8, 6), (8, 6), "attentive_entropy", False, "sgd"),
    "none_noattn": ("none", "none", "none", 1, 5, (8, 6), (8, 6), "attentive_entropy", False, "sgd"),
    "none_pretrain": ("none", "TransAttn", "none", 1, 5, (8, 6), (8, 6), "attentive_entropy", True, "sgd"),
    "none_short": ("none", "TransAttn", "none", 1, 5, (10, 7), (6, 3), "attentive_entropy", False, "sgd"),
    "none_adam": ("none", "none", "none", 1, 5, (8, 6), (8, 6), "attentive_entropy", True, "adam"),
}


@gpu
@pytest.mark.parametrize("case", list(CASES))
def test_three_iterations_match_the_stock_autograd_loop(case):
    """Three iterations against main.py:388-583 under --use_target Sv / none on this repo's VideoModel: autograd,
    loss.ta3n_loss(use_target=...), clip_grad_norm_ over the parameters with a gradient and torch.optim SGD(nesterov)
    / Adam, zero_grad() before each update.  Losses, parameters and the exported optimizer state agree (fp32 engine)."""
    import ta3n_b200
    from ta3n_b200 import loss as LS
    from ta3n_b200.train import Adam, SGDNesterov, TrainStep
    use_target, attn, attn_frame, add_fc, T, (Bs, Bt), (ns, nt), extra, pretrain, kind = CASES[case]
    ta3n_b200.set_gemm_engine("fp32")
    try:
        xs, xt, ls, lt = _inputs(ns, nt, T)
        m_a = _model(T=T, attn=attn, attn_frame=attn_frame, add_fc=add_fc)
        m_b = copy.deepcopy(m_a)
        cfg = SGDNesterov(lr=0.01, clip_gradient=0.5) if kind == "sgd" else Adam(lr=1e-3, clip_gradient=0.5)
        step = TrainStep(m_a, Bs, Bt, BETA, gamma=0.3, optimizer=cfg, pretrain_source=pretrain, add_loss_DA=extra,
                         use_target=use_target, stats=True)
        losses = [step(xs, xt, ls, lt).item() for _ in range(3)]
        torch.cuda.synchronize()
        params = list(m_b.parameters())
        if kind == "sgd":
            opt = torch.optim.SGD(params, 0.01, momentum=0.9, weight_decay=1e-4, nesterov=True)
        else:
            opt = torch.optim.Adam(params, 1e-3, weight_decay=1e-4)
        d = _dev()
        ref = []
        for _ in range(3):
            for pre in ((True, False) if pretrain else (False,)):
                opt.zero_grad(set_to_none=True)
                outs = m_b(xs.to(d), xt.to(d), list(BETA), 0, is_train=True, reverse=False)
                if pre:
                    loss = F.cross_entropy(outs[1], ls.to(d))
                else:
                    loss = LS.ta3n_loss(outs, ls.to(d), 0.3, use_attn=attn, add_loss_DA=extra, use_target=use_target,
                                        label_target=lt.to(d))
                    ref.append(loss.item())
                loss.backward()
                if pre or use_target == "none":
                    # this repo's path is one autograd node: it returns zeros where the reference leaves .grad None
                    for p in params:
                        if p.grad is not None and not p.grad.any():
                            p.grad = None
                torch.nn.utils.clip_grad_norm_([p for p in params if p.grad is not None], 0.5)
                opt.step()
        assert losses == pytest.approx(ref, rel=2e-5)
        pb = dict(m_b.named_parameters())
        for name, p in m_a.named_parameters():
            assert_close(p.detach(), pb[name].detach(), 1e-5, name)
        mine, theirs = step.optimizer_state_dict(), opt.state_dict()
        assert sorted(mine["state"]) == sorted(theirs["state"])
        for i, entry in theirs["state"].items():
            for k, v in entry.items():
                if k == "step":
                    assert float(mine["state"][i][k]) == float(v), (i, k)
                else:
                    assert_close(mine["state"][i][k], v.cpu(), 1e-4, f"state[{i}][{k}]", noise=1e-9)
        # the state loads back, Adam step counts included
        step.load_optimizer_state_dict(theirs)
        again = step.optimizer_state_dict()
        assert {i: float(e["step"]) for i, e in again["state"].items() if "step" in e} == \
            {i: float(e["step"]) for i, e in theirs["state"].items() if "step" in e}
    finally:
        ta3n_b200.set_gemm_engine("tf32x3")


@gpu
@pytest.mark.parametrize("use_target,kind,pretrain", [("Sv", "sgd", False), ("Sv", "adam", True),
                                                      ("none", "sgd", True), ("none", "adam", False)])
def test_eager_graph_reruns_and_resume_are_bit_identical(use_target, kind, pretrain):
    from ta3n_b200.train import Adam, SGDNesterov, TrainStep
    xs, xt, ls, lt = _inputs(8, 6, 5)
    mk = lambda: SGDNesterov(lr=0.01) if kind == "sgd" else Adam(lr=1e-3)           # noqa: E731
    kw = dict(seed=11, gamma=0.3, use_target=use_target, pretrain_source=pretrain)
    runs = []
    for use_graph in (False, True, True):
        step = TrainStep(_model(drop=0.5), 8, 6, BETA, use_graph=use_graph, optimizer=mk(), **kw)
        if use_graph:
            step.step_counter.fill_(0)
        losses = []
        for i in range(3):
            n = (8, 6) if i != 1 else (5, 3)
            losses.append(step(xs[:n[0]], xt[:n[1]], ls[:n[0]], lt[:n[1]]).clone())
        torch.cuda.synchronize()
        runs.append((torch.cat(losses), step.flat_param.clone()))
    for other in runs[1:]:
        assert torch.equal(runs[0][0], other[0]) and torch.equal(runs[0][1], other[1])

    m_a = _model(drop=0.5)
    m_b = copy.deepcopy(m_a)
    a = TrainStep(m_a, 8, 6, BETA, optimizer=mk(), **kw)
    for _ in range(4):
        a(xs, xt, ls, lt)
    b = TrainStep(m_b, 8, 6, BETA, optimizer=mk(), **kw)
    for _ in range(2):
        b(xs, xt, ls, lt)
    sd = copy.deepcopy(b.state_dict())
    params = copy.deepcopy(m_b.state_dict())
    m_c = _model(drop=0.5, seed=99)
    m_c.load_state_dict(params)
    c = TrainStep(m_c, 8, 6, BETA, optimizer=mk(), **kw)
    c.load_state_dict(sd)
    for _ in range(2):
        c(xs, xt, ls, lt)
    torch.cuda.synchronize()
    assert torch.equal(a.flat_param, c.flat_param)


@gpu
def test_target_labels_are_checked():
    from ta3n_b200.train import SGDNesterov, TrainStep
    xs, xt, ls, lt = _inputs(8, 6, 5)
    step = TrainStep(_model(), 8, 6, BETA, optimizer=SGDNesterov(lr=0.01), use_target="Sv")
    with pytest.raises(ValueError, match="target_labels"):
        step(xs, xt, ls)
    with pytest.raises(ValueError, match="target_labels"):
        step(xs, xt, ls, lt[:5])
    with pytest.raises(ValueError, match="target_labels"):
        step.load(xs, xt[:4], ls, lt)


@gpu
@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_usv_is_the_default(kind):
    """use_target='uSv' issues the default step's launches and gives its losses, gradients and parameters bit for
    bit; 'none' issues fewer launches."""
    import ta3n_b200
    from ta3n_b200.train import Adam, SGDNesterov, TrainStep
    from tests.test_discrepancy import PLAIN_LAUNCHES
    ta3n_b200.set_gemm_engine("tf32x3")
    xs, xt, ls, lt = _inputs(8, 6, 5)
    mk = lambda: SGDNesterov(lr=0.01) if kind == "sgd" else Adam(lr=1e-3)           # noqa: E731
    a = TrainStep(_model(drop=0.5), 8, 6, BETA, optimizer=mk(), seed=5, stats=True)
    b = TrainStep(_model(drop=0.5), 8, 6, BETA, optimizer=mk(), seed=5, stats=True, use_target="uSv")
    n = TrainStep(_model(drop=0.5), 8, 6, BETA, optimizer=mk(), seed=5, use_target="none")
    plain = TrainStep(_model(drop=0.5), 8, 6, BETA, optimizer=mk(), seed=5)
    assert a.launches_per_step == b.launches_per_step
    if kind == "sgd":
        assert plain.launches_per_step == PLAIN_LAUNCHES[True]
    assert n.launches_per_step < plain.launches_per_step
    for _ in range(3):
        la, lb = a(xs, xt, ls).clone(), b(xs, xt, ls, lt).clone()
        torch.cuda.synchronize()
        assert torch.equal(la, lb)
        assert torch.equal(a.flat_grad, b.flat_grad) and torch.equal(a.flat_param, b.flat_param)
    assert torch.equal(a.stats_acc, b.stats_acc)


@gpu
@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_none_leaves_the_parameters_outside_p_alone(kind):
    """Under 'none' the parameters the CE never reaches (the video discriminator; the relation discriminators
    without attention; the frame discriminator without frame attention) keep their values bit for bit, with weight
    decay on, and their gradient slots stay zero; the loss is the source CE the step reports."""
    from ta3n_b200.train import Adam, SGDNesterov, TrainStep
    xs, xt, ls, lt = _inputs(8, 6, 5)
    m = _model(attn="none")
    before = {k: v.detach().clone() for k, v in m.named_parameters()}
    opt = SGDNesterov(lr=0.05, weight_decay=1e-2) if kind == "sgd" else Adam(lr=1e-2, weight_decay=1e-2)
    step = TrainStep(m, 8, 6, BETA, optimizer=opt, use_target="none")
    for _ in range(4):
        step(xs, xt, ls)
    torch.cuda.synchronize()
    moved = {k for k, v in m.named_parameters() if not torch.equal(v.detach(), before[k])}
    idle = {k for k in before if k.startswith(("fc_feature_domain", "fc_classifier_domain", "relation_domain_"))
            or "domain" in k}
    assert idle and not (moved & idle), moved & idle
    assert "fc_classifier_video_source.weight" in moved
    for k, p in m.named_parameters():
        if k in idle and p.grad is not None:
            assert not p.grad.any(), k


@gpu
@pytest.mark.parametrize("use_target", ["Sv", "none"])
def test_meters(use_target):
    """stats() against AverageMeters fed main.py's values from the step's own logits: Sv folds the CE and top-k over
    source and target rows with n = the real source rows; none keeps loss, loss_c and top-k over the source rows and
    leaves loss_a / loss_e / loss_s at count 0."""
    from oracle.train_stats_oracle import AverageMeter
    from ta3n_b200.train import SGDNesterov, TrainStep
    Bs, Bt = 8, 6
    xs, xt, ls, lt = _inputs(Bs, Bt, 5)
    step = TrainStep(_model(drop=0.5), Bs, Bt, BETA, optimizer=SGDNesterov(lr=0.01), stats=True, use_target=use_target)
    ml, mc, m1 = AverageMeter(), AverageMeter(), AverageMeter()
    for ns, nt in ((8, 6), (8, 6), (5, 2)):
        loss = step(xs[:ns], xt[:nt], ls[:ns], lt[:nt]).item()
        pv = step.outputs[5].cpu()
        if use_target == "Sv":
            z, y = torch.cat([pv[:ns], pv[Bs:Bs + nt]]).double(), torch.cat([ls[:ns], lt[:nt]])
        else:
            z, y = pv[:ns].double(), ls[:ns]
        ml.update(loss)
        mc.update(F.cross_entropy(z, y).item(), ns)
        m1.update(100.0 * (z.argmax(1) == y).sum().item() / z.shape[0], ns)
    st = step.stats()
    snap = step.stats_async().result()
    assert st.loss.count == 3 and st.loss.avg == pytest.approx(ml.avg, rel=1e-6)
    assert st.loss_c.count == 21 and st.loss_c.avg == pytest.approx(mc.avg, rel=1e-5)
    assert st.top1.count == 21 and st.top1.avg == pytest.approx(m1.avg, rel=1e-9)
    assert snap.top1 == st.top1 and snap.loss_c == st.loss_c
    if use_target == "none":
        assert st.loss_a.count == st.loss_e.count == st.loss_s.count == 0
    else:
        assert st.loss_a.count > 0 and st.loss_e.count == 14
    step.reset_stats()
    assert step.stats().top1.count == 0 and step.stats().top1.sum == 0.0


@gpu
def test_device_sampler_and_double_buffer_carry_the_target_labels(tmp_path):
    """Under Sv the sampler-fed step equals the load()-fed one bit for bit over two epochs with short last batches,
    and double_buffer + prefetch equals the single-slot step."""
    from ta3n_b200 import dataset as D
    from ta3n_b200.train import SGDNesterov, TrainStep
    from tests.test_device_sampler import _banks
    T, batch = 5, (8, 6)
    sets, banks = _banks(tmp_path, T, orc.FEATURE_DIM, (21, None), (9, 14), batch)
    model_a = _model(drop=0.5)
    model_b = copy.deepcopy(model_a)
    kw = dict(beta=BETA, gamma=0.3, seed=123, use_target="Sv", stats=True)
    sampler = D.DevicePairedSampler(banks[0], banks[1], batch, seed=4)
    step_a = TrainStep(model_a, *batch, sampler=sampler, optimizer=SGDNesterov(lr=0.01), **kw)
    step_b = TrainStep(model_b, *batch, optimizer=SGDNesterov(lr=0.01), **kw)
    loader = D.PairedFeatureLoader(sets[0], sets[1], batch, seed=4)
    n_step = 0
    for epoch in range(2):
        assert sampler.start_epoch() == len(loader) == 3
        for (xs, ys), (xt, yt) in loader:
            if xs.shape[0] < batch[0] or xt.shape[0] < batch[1]:
                step_b.xs.zero_(), step_b.xt.zero_(), step_b.labels.zero_(), step_b.labels_t.zero_()
            step_b.load(xs, xt, ys, yt)
            loss_b = step_b.run().clone()
            loss_a = step_a.run().clone()
            torch.cuda.synchronize()
            n_step += 1
            assert torch.equal(step_a.labels_t, step_b.labels_t), (epoch, n_step)
            assert torch.equal(loss_a, loss_b) and torch.equal(step_a.flat_param, step_b.flat_param), (epoch, n_step)
    assert n_step == 6
    assert torch.equal(step_a.stats_acc, step_b.stats_acc) and torch.equal(step_a.prec_sum, step_b.prec_sum)

    xs, xt, ls, lt = _inputs(8, 6, 5)
    m_a = _model(drop=0.5)
    m_b = copy.deepcopy(m_a)
    a = TrainStep(m_a, 8, 6, BETA, optimizer=SGDNesterov(lr=0.01), seed=7, use_target="Sv")
    b = TrainStep(m_b, 8, 6, BETA, optimizer=SGDNesterov(lr=0.01), seed=7, use_target="Sv", double_buffer=True)
    a.step_counter.fill_(0)
    b.step_counter.fill_(0)
    b.load(xs, xt, ls, lt)
    for i in range(3):
        lt_i = (lt + i) % 7
        a(xs, xt, ls, lt_i)
        b.run()
        if i < 2:
            b.prefetch(xs, xt, ls, (lt + i + 1) % 7)
            b.swap()
    torch.cuda.synchronize()
    assert torch.equal(a.flat_param, b.flat_param)


@gpu
def test_none_with_overlap_allreduce_on_one_rank():
    """overlap_allreduce=True on one rank asks for a bucket split; the source-only pass has none, so the step is one
    graph and equals the step without the option."""
    from ta3n_b200.train import SGDNesterov, TrainStep
    xs, xt, ls, _ = _inputs(8, 6, 5)
    m_a = _model(drop=0.5)
    m_b = copy.deepcopy(m_a)
    a = TrainStep(m_a, 8, 6, BETA, optimizer=SGDNesterov(lr=0.01), seed=3, use_target="none", overlap_allreduce=True)
    b = TrainStep(m_b, 8, 6, BETA, optimizer=SGDNesterov(lr=0.01), seed=3, use_target="none")
    assert not a.split and a.graphs[0][1] is None
    for _ in range(2):
        a(xs, xt, ls)
        b(xs, xt, ls)
    torch.cuda.synchronize()
    assert torch.equal(a.flat_param, b.flat_param)
