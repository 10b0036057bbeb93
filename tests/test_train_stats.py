"""The training meters on the device: the kernel (C ABI ta3n_train_stats_accumulate) and TrainStep(stats=True).

CPU: the fp64 restatement of main.py's meter arithmetic (oracle/train_stats_oracle.py) against the reference's train()
(tests/golden/train_stats_golden.npz), the accumulator's parsing, the C ABI's argument checks, the refusals.
GPU: the kernel alone on planted logits at fp32 grade; TrainStep's meters against the fp64 restatement on the logits
the step produced, against the reference's epoch (host pipeline and device sampler), with an optimizer, and without
any effect on the step's results.

fp32 grade, per term:  |cuda - ref64| <= TOL_FP32 * |ref64| + 8 * noise,  noise = max(|ref32 - ref64|, 4 ulp * |ref64|).
"""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from oracle import gen_golden_train_stats as gen
from oracle import train_stats_oracle as tso
from tests.golden_util import TOL_FP32, TOL_PATH

gpu = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
LOSS_METERS = ("loss", "loss_c", "loss_a", "loss_e", "loss_s")
ULP = 2.0 ** -23


def _golden():
    z = np.load(os.path.join(HERE, "golden", "train_stats_golden.npz"))
    return z, json.loads(bytes(z["meta_json"]).decode())


def _entropy_on(c):
    return c["add_loss_DA"] == "attentive_entropy" and c["use_attn"] != "none"


def _fixture_step(z, case, i):
    """The reference's removeDummy'd outputs of step i as the oracle's 10-tuple, and pass 2 under MCD."""
    k = f"{case}/step{i}/"
    pd_s = [z[k + f"pd_s{lvl}"] for lvl in range(3)]
    pd_t = [z[k + f"pd_t{lvl}"] for lvl in range(3)]
    outs = (None, z[k + "out_s"], z[k + "out_s_2"], pd_s, None, None, z[k + "out_t"], None, pd_t, None)
    pass2 = (z[k + "out_t_p2"], z[k + "out_t_2_p2"]) if k + "out_t_p2" in z.files else None
    return outs, pass2


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(gen.CASES))
def test_oracle_reproduces_reference_meters(case):
    """Every step's (val, n) of every meter of the reference's train(), and the epoch's AverageMeters, from the fp64
    restatement on the reference's own outputs (the reference computes in fp32: 1e-5)."""
    z, _ = _golden()
    c = gen.CASES[case]
    _, labels, _, cw, dw = gen.case_inputs(c)
    ref = z[case + "/steps"]
    steps = []
    for i, (idx_s, idx_t) in enumerate(gen.case_batches(c)):
        outs, pass2 = _fixture_step(z, case, i)
        st = tso.step_meters(outs, labels[idx_s].numpy(), len(idx_s), len(idx_t), place_adv=c["place_adv"],
                             attentive_entropy=_entropy_on(c), class_weight=cw, domain_weight=dw, pass2=pass2,
                             gamma=gen.GAMMA)
        steps.append(st)
        for j, m in enumerate(gen.METERS):
            if m.startswith("top"):
                q = (1, 5).index(int(m[3:]))
                val, n = 100.0 * st["correct"][q] / st["rows"], st["rows"]
                assert abs(val - ref[i, j, 0]) <= 1e-4, (case, i, m)
                assert n == ref[i, j, 1]
                continue
            if st[m] is None:
                assert np.isnan(ref[i, j]).all(), (case, i, m)
                continue
            val, n = st[m]
            assert n == ref[i, j, 1], (case, i, m, n, ref[i, j, 1])
            assert abs(val - ref[i, j, 0]) <= 1e-5 * abs(ref[i, j, 0]) + 1e-6, (case, i, m, val, ref[i, j, 0])
    ep = z[case + "/epoch"]
    meters = tso.fold(steps)
    for j, m in enumerate(gen.METERS):
        mt = meters[m]
        assert mt.count == ep[j, 3], (case, m)
        for got, want in ((mt.val, ep[j, 0]), (mt.avg, ep[j, 1]), (mt.sum, ep[j, 2])):
            assert abs(got - want) <= 1e-5 * abs(want) + 1e-5, (case, m, got, want)


def test_oracle_tie_rule_and_degenerate_rows():
    """Ties rank by class index; a NaN logit or a label outside [0, C) is a hit at no k and a NaN CE."""
    zz = np.array([[1.0, 3.0, 3.0, 0.0, 3.0], [2.0, 2.0, 2.0, 2.0, 2.0], [np.nan, 0, 0, 0, 0], [0, 1, 2, 3, 4]])
    y = np.array([2, 4, 0, 7])
    assert tso.label_rank(zz, y).tolist() == [1, 4, tso.UNRANKED, tso.UNRANKED]
    ce, ok = tso._ce_rows(zz, y)
    assert np.isnan(ce[2]) and np.isnan(ce[3]) and ok.tolist() == [True, True, True, False]


def test_parse_train_stats():
    """The accumulator's words as AverageMeters: avg = sum / count, 0 while count is 0; precision val from the last
    step's counts, sum = 100 * correct."""
    from ta3n_b200.train import parse_train_stats
    w = np.zeros(27, dtype=np.int64)
    f = w.view(np.float64)
    f[0:5] = [6.0, 10.0, 0.0, 3.0, 0.0]          # sums
    f[5:10] = [2.5, 1.5, 0.0, 0.25, 0.0]         # vals
    w[10:15] = [3, 8, 0, 4, 0]                   # counts
    w[15:17] = [5, 7]                            # correct over the epoch (k = 1, 3)
    w[19:21] = [1, 2]                            # correct of the last step
    w[23], w[24], w[25] = 8, 4, 3                # rows, rows of the last step, steps
    st = parse_train_stats(w, (1, 3))
    assert (st.loss.val, st.loss.avg, st.loss.sum, st.loss.count) == (2.5, 2.0, 6.0, 3)
    assert st.loss_c.avg == 10.0 / 8 and st.loss_a.count == 0 and st.loss_a.avg == 0.0
    assert st.top1.val == 25.0 and st.top1.avg == 62.5 and st.top1.count == 8 and st.top1.sum == 500.0
    assert st.prec[3].val == 50.0 and st.prec[3].avg == 87.5 and st.top5 is None
    assert st.steps == 3 and st.rows == 8 and st.correct == (5, 7)


@pytest.fixture(scope="module")
def lib():
    from ta3n_b200 import build
    build.build()
    from ta3n_b200 import _lib
    return _lib.load()


def test_train_stats_validates_arguments_without_gpu(lib):
    """Null accumulator, top-k values outside [1, C] or more than four, no rows, bad flags, a lone MCD input and a
    short workspace are refused on the host, before any CUDA call."""
    k2 = (C.c_int * 2)(1, 5)
    dw = (C.c_float * 2)(1.0, 1.0)
    ws = 1 << 12

    def call(**kw):
        a = dict(pv=16, lab=32, rel=48, dom=64, frame=80, p2s=None, p2t=None, loss=96, Bs=4, Bt=4, T=5, R=4, C=12,
                 flags=15, valid=None, cw=None, dw=dw, n_k=2, k=k2, acc=4096, ws=8192, ws_bytes=ws)
        a.update(kw)
        return lib.ta3n_train_stats_accumulate(a["pv"], a["lab"], a["rel"], a["dom"], a["frame"], a["p2s"], a["p2t"],
                                               a["loss"], a["Bs"], a["Bt"], a["T"], a["R"], a["C"], a["flags"],
                                               a["valid"], a["cw"], a["dw"], a["n_k"], a["k"], a["acc"], a["ws"],
                                               a["ws_bytes"], None)

    assert call(acc=None) == 1 and b"null accumulator" in lib.ta3n_last_error()
    assert call(k=(C.c_int * 2)(1, 13)) == 1 and b"outside [1, C=12]" in lib.ta3n_last_error()
    assert call(k=(C.c_int * 2)(0, 5)) == 1
    assert call(n_k=5, k=(C.c_int * 5)(1, 2, 3, 4, 5)) == 1 and b"top-k" in lib.ta3n_last_error()
    assert call(n_k=0) == 1
    assert call(Bs=0, Bt=0) == 1 and b"bad sizes" in lib.ta3n_last_error()
    assert call(Bs=0) == 1
    assert call(flags=16) == 1 and b"flags" in lib.ta3n_last_error()
    assert call(flags=-1) == 1
    assert call(p2s=112) == 1 and b"pred2_s without pred2_t" in lib.ta3n_last_error()
    assert call(p2t=112) == 1 and b"pred2_t without pred2_s" in lib.ta3n_last_error()
    assert call(pv=None) == 1
    assert call(acc=4100) == 1 and b"8-byte aligned" in lib.ta3n_last_error()
    assert call(ws_bytes=16) == 2 and b"workspace too small" in lib.ta3n_last_error()
    assert lib.ta3n_train_stats_workspace_bytes(0) == 0 and lib.ta3n_train_stats_workspace_bytes(9) > 0


def _cpu_model(**kw):
    from ta3n_b200.models import VideoModel
    return VideoModel(5, "video", "trn-m", "RGB", train_segments=5, val_segments=5, fc_dim=64, verbose=False,
                      **kw).train()


def test_train_step_stats_refuses_several_ranks(monkeypatch):
    from ta3n_b200 import train
    monkeypatch.setattr(train.dist, "is_initialized", lambda: True)
    monkeypatch.setattr(train.dist, "get_world_size", lambda group=None: 2)
    with pytest.raises(NotImplementedError, match="single rank"):
        train.TrainStep(_cpu_model(), 4, 4, beta=[0.75, 0.75, 0.5], stats=True)


# ------------------------------------------------------------------------------------------------
# GPU: the kernel alone
# ------------------------------------------------------------------------------------------------
def _abi_outs(pv, labels, rel, dom, frame, Bs, T, p2s=None, p2t=None):
    """C-ABI layout (M rows, source first) -> the oracle's 10-tuple and pass 2 (numpy, fp64)."""
    f = lambda t: t.detach().double().cpu().numpy()          # noqa: E731
    pv, rel, dom, frame = f(pv), f(rel), f(dom), f(frame).reshape(pv.shape[0], T, 2)
    s2 = f(p2s) if p2s is not None else None
    pd_s, pd_t = [rel[:Bs], dom[:Bs], frame[:Bs]], [rel[Bs:], dom[Bs:], frame[Bs:]]
    outs = (None, pv[:Bs], s2, pd_s, None, None, pv[Bs:], None, pd_t, None)
    pass2 = (pv[Bs:], f(p2t)) if p2t is not None else None
    return outs, pass2


def _meters_at(outs, labels, vs, vt, place_adv, entropy, cw, dw, pass2, topk):
    kw = dict(place_adv=place_adv, attentive_entropy=entropy, class_weight=cw, domain_weight=dw, pass2=pass2,
              gamma=0.003, topk=topk)
    return tso.step_meters(outs, labels, vs, vt, **kw), tso.step_meters(outs, labels, vs, vt, dtype=np.float32, **kw)


def _assert_fp32_grade(got, r64, r32, what):
    noise = max(abs(r32 - r64), 4 * ULP * abs(r64))
    assert abs(got - r64) <= TOL_FP32 * abs(r64) + 8 * noise, f"{what}: {got!r} vs {r64!r} (noise {noise:.2e})"


def _acc_words(acc, pad):
    return acc[pad:pad + 27].cpu().numpy()


def _run_kernel(lib, inputs, Bs, Bt, T, R, Cc, flags, valid, cw, dw, ks, acc, ws, mcd):
    pv, labels, rel, dom, frame, p2s, p2t, loss = inputs
    P = lambda t: None if t is None else t.data_ptr()       # noqa: E731
    k = (C.c_int * len(ks))(*ks)
    dwc = (C.c_float * 2)(*dw)
    rc = lib.ta3n_train_stats_accumulate(P(pv), P(labels), P(rel), P(dom), P(frame), P(p2s) if mcd else None,
                                         P(p2t) if mcd else None, P(loss), Bs, Bt, T, R, Cc, flags, P(valid), P(cw),
                                         dwc, len(ks), k, acc.data_ptr(), P(ws), ws.numel(), None)
    assert rc == 0, lib.ta3n_last_error()


def _planted(Bs, Bt, T, Cc, seed, dev):
    g = torch.Generator().manual_seed(seed)
    M, R = Bs + Bt, T - 1
    pv = torch.randn(M, Cc, generator=g) * 2
    labels = torch.randint(0, Cc, (Bs,), generator=g)
    # ties at the top-k boundary: the label's logit equals the values around ranks 1 and 5
    for r in range(0, Bs, 5):
        srt = torch.sort(pv[r], descending=True).values
        pv[r, labels[r]] = srt[min(4, Cc - 1)] if r % 2 else srt[0]
    # degenerate rows among the last three source rows: real in the first (full) step only
    if Bs > 7:
        pv[Bs - 1, :] = float("-inf")                          # every class ties
        pv[Bs - 2, Cc // 2] = float("nan")                     # unranked, NaN CE
        labels[Bs - 3] = Cc + 2                                # outside [0, C)
    rel = torch.randn(M, R, 2, generator=g)
    dom = torch.randn(M, 2, generator=g)
    frame = torch.randn(M * T, 2, generator=g)
    p2s = torch.randn(Bs, Cc, generator=g)
    p2t = torch.randn(Bt, Cc, generator=g)
    loss = torch.tensor([1.2345678])
    return [t.to(dev) for t in (pv, labels, rel, dom, frame, p2s, p2t, loss)]


@gpu
@pytest.mark.parametrize("mcd,weighted", [(False, False), (True, False), (False, True)])
@pytest.mark.parametrize("Cc,Bs,Bt,T", [(5, 13, 11, 5), (12, 40, 30, 3), (33, 9, 0, 10), (1000, 17, 6, 5),
                                        (5, 1100, 1000, 4)])
def test_kernel_against_fp64(lib, Cc, Bs, Bt, T, mcd, weighted):
    """Three steps into one accumulator -- all rows real, a short batch, no real target row -- against the fp64
    restatement per term at fp32 grade; top-k counts exactly (with planted ties, NaN / -inf rows and a label outside
    [0, C) when the batch has room); NaN terms only where the oracle has them; the guard words around the
    accumulator untouched; a rerun bit-identical.  M = 2100 spans more than 256 CTAs (two passes of the fold)."""
    dev = torch.device("cuda")
    R = T - 1
    inputs = _planted(Bs, Bt, T, Cc, 7 + Cc + Bs, dev)
    labels_np = inputs[1].cpu().numpy()
    g = torch.Generator().manual_seed(3)
    cw = (0.5 + torch.rand(Cc, generator=g)).to(dev) if weighted else None
    dw = (0.7, 1.3) if weighted else (1.0, 1.0)
    ks = (1, 5, Cc) if Cc >= 5 else (1,)
    flags = 15
    place = ("Y", "Y", "Y")
    pad = 4
    ws = torch.zeros(max(256, lib.ta3n_train_stats_workspace_bytes(Bs + Bt)), device=dev, dtype=torch.uint8)
    plans = [(Bs, Bt), (max(1, Bs - 3), max(0, Bt - 2)), (max(1, Bs // 2), 0)]

    def epoch():
        acc = torch.full((27 + 2 * pad,), -7, device=dev, dtype=torch.int64)
        acc[pad:pad + 27] = 0
        valid = torch.zeros(2, device=dev, dtype=torch.int32)
        snaps = []
        for vs, vt in plans:
            valid.copy_(torch.tensor([vs, vt], dtype=torch.int32))
            _run_kernel(lib, inputs, Bs, Bt, T, R, Cc, flags, valid, cw, dw, ks, acc[pad:], ws, mcd)
            snaps.append(_acc_words(acc, pad).copy())
        assert torch.all(acc[:pad] == -7) and torch.all(acc[pad + 27:] == -7)
        return snaps

    snaps = epoch()
    again = epoch()
    for a, b in zip(snaps, again):
        assert np.array_equal(a, b)                              # bit-identical rerun
    from ta3n_b200.train import parse_train_stats
    pv, _, rel, dom, frame, p2s, p2t, loss = inputs
    outs, pass2 = _abi_outs(pv, labels_np, rel, dom, frame, Bs, T, p2s if mcd else None, p2t if mcd else None)
    steps = []
    cw_np = None if cw is None else cw.cpu().numpy()
    for (vs, vt), words in zip(plans, snaps):
        st = parse_train_stats(words, ks)
        r64, r32 = _meters_at(outs, labels_np, vs, vt, place, True, cw_np, np.array(dw), pass2, ks)
        steps.append(r64)
        assert st.loss.val == float(np.float32(1.2345678))
        for m in ("loss_c", "loss_a", "loss_e", "loss_s"):
            meter = getattr(st, m)
            if r64[m] is None:
                assert meter.count == 0, m
                continue
            val, n = r64[m]
            if np.isnan(val):
                assert np.isnan(meter.val), m
            else:
                _assert_fp32_grade(meter.val, val, r32[m][0], f"C={Cc} vs={vs} vt={vt} {m}")
        assert words[24] == vs
        assert tuple(int(c) for c in words[19:19 + len(ks)]) == r64["correct"], (vs, vt)
    st = parse_train_stats(snaps[-1], ks)
    ref = tso.fold(steps, topk=ks)
    assert st.steps == 3 and st.rows == sum(p[0] for p in plans)
    for m in ("loss_c", "loss_a", "loss_e", "loss_s"):
        assert getattr(st, m).count == ref[m].count, m
    assert st.loss_s.count == (sum(p[1] for p in plans) if mcd else 0)
    assert st.correct == tuple(sum(s["correct"][q] for s in steps) for q in range(len(ks)))


@gpu
def test_kernel_terms_switched_off_keep_count_zero(lib):
    """No adversarial level, no entropy, no MCD: only loss, loss_c and the precision meters move."""
    dev = torch.device("cuda")
    Bs, Bt, T, Cc = 10, 6, 5, 7
    inputs = _planted(Bs, Bt, T, Cc, 11, dev)
    acc = torch.zeros(27, device=dev, dtype=torch.int64)
    ws = torch.zeros(max(256, lib.ta3n_train_stats_workspace_bytes(Bs + Bt)), device=dev, dtype=torch.uint8)
    for flags in (0, 1, 2, 4):
        acc.zero_()
        _run_kernel(lib, inputs, Bs, Bt, T, T - 1, Cc, flags, None, None, (1.0, 1.0), (1, 5), acc, ws, False)
        w = acc.cpu().numpy()
        counts = w[10:15]
        n_a = {0: 0, 1: (Bs + Bt) * (T - 1), 2: Bs + Bt, 4: (Bs + Bt) * T}[flags]
        assert counts.tolist() == [1, Bs, n_a, 0, 0], flags


# ------------------------------------------------------------------------------------------------
# GPU: TrainStep
# ------------------------------------------------------------------------------------------------
def _gpu_model(C_=7, T=5, use_attn="TransAttn", attn_frame="none", mcd=False, seed=0):
    from ta3n_b200.models import VideoModel
    torch.manual_seed(seed)
    kw = dict(ens_DA="MCD") if mcd else {}
    m = VideoModel(C_, "video", "trn-m", "RGB", train_segments=T, val_segments=T, fc_dim=128, use_attn=use_attn,
                   use_attn_frame=attn_frame, dropout_i=0.0, dropout_v=0.0, verbose=False, **kw).cuda().train()
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():                                   # spread the predictions over the classes
        for n, p in m.named_parameters():
            if "weight" in n:
                p.add_(0.05 * torch.randn(p.shape, generator=g).to(p.device))
    return m


VARIANTS = {
    "T3": dict(T=3),
    "T5": dict(T=5),
    "T10": dict(T=10),
    "none": dict(use_attn="none"),
    "attn_frame": dict(attn_frame="TransAttn", legacy_only=True),
    "mcd_mu0": dict(mcd=True, mu=0.0, legacy_only=True),
    "mcd_mu07": dict(mcd=True, mu=0.7, legacy_only=True),
    "weights": dict(weighted=True, phased_only=True),
    "adv_YYN": dict(place_adv="YYN"),
    "adv_NYN": dict(place_adv="NYN", add_loss_DA="none"),
    "adv_YNN": dict(place_adv="YNN", add_loss_DA="none"),
}
PARAMS = [(v, mode, eng) for v, o in VARIANTS.items() for mode in ("legacy", "phased")
          if not (o.get("legacy_only") and mode == "phased") and not (o.get("phased_only") and mode == "legacy")
          for eng in ("fp32", "tf32x3")]


def _make_step(model, Bs, Bt, o, mode, **kw):
    from ta3n_b200.train import TrainStep
    C_ = model.fc_classifier_video_source.weight.shape[0]
    g = torch.Generator().manual_seed(5)
    cw = (0.5 + torch.rand(C_, generator=g)) if o.get("weighted") else None
    dw = (0.7, 1.3) if o.get("weighted") else (1.0, 1.0)
    beta = [0.75, -1.0, 0.5] if o.get("weighted") else [0.75, 0.75, 0.5]
    step = TrainStep(model, Bs, Bt, beta=beta, gamma=0.003, place_adv=tuple(o.get("place_adv", "YYY")),
                     add_loss_DA=o.get("add_loss_DA", "attentive_entropy"), mode=mode, class_weight=cw,
                     domain_weight=dw, mu=o.get("mu", 0.0), **kw)
    if o.get("weighted"):
        step.set_progress(0.3)
    return step, cw, dw


def _step_oracle(step, o, labels, vs, vt, cw, dw, dtype=np.float64):
    """The fp64 restatement on the logits the step just produced (step.outputs)."""
    out = step.outputs
    Bs, T = step.Bs, step.T
    pv, rel, dom, frame = out[5], out[3], out[6], out[1]
    outs, pass2 = _abi_outs(pv, labels, rel, dom, frame.reshape(-1, 2), Bs, T,
                            step.pred2_s if step.mcd else None, step.pred2_t if step.mcd else None)
    entropy = bool(step.flags & 8)
    return tso.step_meters(outs, labels, vs, vt, place_adv=o.get("place_adv", "YYY"), attentive_entropy=entropy,
                           class_weight=None if cw is None else cw.numpy(), domain_weight=np.array(dw), pass2=pass2,
                           gamma=0.003, dtype=dtype)


@gpu
@pytest.mark.parametrize("variant,mode,engine", PARAMS)
def test_train_step_meters_match_oracle_on_its_logits(variant, mode, engine):
    """Two steps (the second a short batch) with stats=True, no optimizer: each term's val matches the fp64
    restatement on the logits the step produced at fp32 grade, the top-k counts exactly, the loss meter is the loss
    buffer, and loss_c + loss_a + gamma loss_e + loss_s equals the step's loss to fp32 rounding."""
    import ta3n_b200
    ta3n_b200.set_gemm_engine(engine)
    o = VARIANTS[variant]
    T = o.get("T", 5)
    model = _gpu_model(T=T, use_attn=o.get("use_attn", "TransAttn"), attn_frame=o.get("attn_frame", "none"),
                       mcd=o.get("mcd", False))
    Bs, Bt = 9, 7
    step, cw, dw = _make_step(model, Bs, Bt, o, mode, stats=True)
    g = torch.Generator().manual_seed(17)
    try:
        for vs, vt in ((Bs, Bt), (5, 3)):
            xs, xt = torch.randn(vs, T, 2048, generator=g), torch.randn(vt, T, 2048, generator=g) + 0.2
            y = torch.randint(0, 7, (vs,), generator=g)
            step.xs.zero_(), step.xt.zero_(), step.labels.zero_()
            loss = step(xs, xt, y).item()
            st = step.stats()
            r64 = _step_oracle(step, o, y.numpy(), vs, vt, cw, dw)
            r32 = _step_oracle(step, o, y.numpy(), vs, vt, cw, dw, dtype=np.float32)
            assert st.loss.val == loss
            total = 0.0
            for m in ("loss_c", "loss_a", "loss_e", "loss_s"):
                meter = getattr(st, m)
                if r64[m] is None:
                    assert meter.count == 0, m
                    continue
                _assert_fp32_grade(meter.val, r64[m][0], r32[m][0], f"{variant} {mode} {engine} {m}")
                total += meter.val * (0.003 if m == "loss_e" else 1.0)
            assert abs(total - loss) <= 32 * ULP * (abs(st.loss_c.val) + abs(st.loss_a.val) + abs(st.loss_s.val) + 1)
            assert tuple(round(m.val * vs / 100) for m in (st.top1, st.top5)) == r64["correct"]
        assert st.steps == 2 and st.rows == Bs + 5 and st.loss.count == 2
    finally:
        ta3n_b200.set_gemm_engine("tf32x3")


def _shards(tmp_path, c, xs, labels, xt):
    from ta3n_b200 import dataset as D
    paths = []
    for name, x, y in (("src", xs, labels), ("tgt", xt, torch.zeros(xt.shape[0], dtype=torch.int64))):
        path = os.path.join(str(tmp_path), name + ".npy")
        np.save(path, x.numpy().astype(np.float32))
        with open(path + ".json", "w") as f:
            json.dump({"num_segments": c["T"], "labels": [int(v) for v in y]}, f)
        paths.append(D.PackedTSNDataSet(path))
    return paths


def _case_model(case, meta):
    from ta3n_b200.models import VideoModel
    c = gen.CASES[case]
    m = VideoModel(c["C"], "video", "trn-m", "RGB", train_segments=c["T"], val_segments=c["T"], fc_dim=c["F"],
                   use_attn=c["use_attn"], ens_DA=c["ens"], dropout_i=0.0, dropout_v=0.0, verbose=False)
    m.load_state_dict(gen.case_params(c, meta[case + "/param_order"]))
    return m.cuda().train()


def _check_epoch_against_fixture(st, z, case):
    ep = z[case + "/epoch"]
    for j, m in enumerate(gen.METERS):
        meter = getattr(st, m)
        assert meter.count == ep[j, 3], (case, m, meter.count, ep[j, 3])
        if m.startswith("top"):
            assert abs(meter.avg - ep[j, 1]) <= 1e-4 and abs(meter.val - ep[j, 0]) <= 1e-4, (case, m)
            continue
        for got, want in ((meter.val, ep[j, 0]), (meter.avg, ep[j, 1])):
            assert abs(got - want) <= TOL_PATH * abs(want) + 1e-6, (case, m, got, want)


@gpu
@pytest.mark.parametrize("pipeline", ["host", "device"])
@pytest.mark.parametrize("case", list(gen.CASES))
def test_train_step_epoch_against_reference(tmp_path, case, pipeline):
    """An epoch at fixed weights (no optimizer) with stats=True against the reference's train(): every meter's val
    and avg within the path budget, every count exactly.  host: prefetch() / swap() of the fixture's batches, the
    short last one included; device: DevicePairedSampler over shards of the same rows, seeded alike."""
    from ta3n_b200 import dataset as D
    c = gen.CASES[case]
    if pipeline == "device" and c["empty_target"]:
        pytest.skip("a paired loader never ends an epoch with an empty target batch")
    z, meta = _golden()
    model = _case_model(case, meta)
    xs, labels, xt, cw, dw = gen.case_inputs(c)
    mode = "phased" if c["weighted"] else "legacy"
    batch = (c["bs"], c["bt"])
    from ta3n_b200.train import TrainStep
    kw = dict(beta=list(gen.BETA), gamma=gen.GAMMA, place_adv=tuple(c["place_adv"]), add_loss_DA=c["add_loss_DA"],
              mode=mode, class_weight=cw, domain_weight=tuple(dw.tolist()) if dw is not None else (1.0, 1.0),
              mu=c["mu"], stats=True)
    if pipeline == "device":
        src, tgt = _shards(tmp_path, c, xs, labels, xt)
        sampler = D.DevicePairedSampler(D.DeviceFeatureBank(src), D.DeviceFeatureBank(tgt), batch,
                                        seed=gen.SAMPLER_SEED)
        step = TrainStep(model, *batch, sampler=sampler, **kw)
        n = sampler.start_epoch()
        assert n == len(gen.case_batches(c))
        for _ in range(n):
            step.run()
    else:
        step = TrainStep(model, *batch, double_buffer=True, **kw)
        plan = gen.case_batches(c)
        idx_s, idx_t = plan[0]
        step.load(xs[idx_s], xt[idx_t], labels[idx_s])
        for i in range(len(plan)):
            if i + 1 < len(plan):
                ns, nt = plan[i + 1]
                step.prefetch(xs[ns], xt[nt], labels[ns])
            step.run()
            if i + 1 < len(plan):
                step.swap()
    _check_epoch_against_fixture(step.stats(), z, case)


@gpu
@pytest.mark.parametrize("opt", ["sgd", "adam"])
@pytest.mark.parametrize("mode", ["legacy", "phased"])
def test_meters_with_an_optimizer_follow_the_weights_before_each_step(opt, mode):
    """With an optimizer each step's vals are those of the weights before its update: the fp64 restatement on
    VideoModel.forward at those weights (fp32 engine), within 1e-4."""
    import ta3n_b200
    from ta3n_b200.train import Adam, SGDNesterov
    ta3n_b200.set_gemm_engine("fp32")
    try:
        model = _gpu_model()
        Bs, Bt, T = 8, 6, 5
        o = {}
        optim = SGDNesterov(lr=0.01) if opt == "sgd" else Adam(lr=1e-3)
        step, cw, dw = _make_step(model, Bs, Bt, o, mode, stats=True, optimizer=optim)
        g = torch.Generator().manual_seed(23)
        for i in range(3):
            xs, xt = torch.randn(Bs, T, 2048, generator=g), torch.randn(Bt, T, 2048, generator=g) + 0.2
            y = torch.randint(0, 7, (Bs,), generator=g)
            with torch.no_grad():
                outs = model(xs.cuda(), xt.cuda(), [0.75, 0.75, 0.5], 0, is_train=True, reverse=False)
            ref = tso.step_meters(outs, y.numpy(), Bs, Bt, class_weight=None, gamma=0.003)
            before = step.flat_param.clone()
            step(xs, xt, y)
            st = step.stats()
            assert not torch.equal(before, step.flat_param)      # the update ran
            for m in ("loss_c", "loss_a", "loss_e"):
                assert abs(getattr(st, m).val - ref[m][0]) <= 1e-4 * abs(ref[m][0]) + 1e-6, (i, m)
            assert abs(st.loss.val - ref["loss"][0]) <= 1e-4 * abs(ref["loss"][0])
        assert st.steps == 3
    finally:
        ta3n_b200.set_gemm_engine("tf32x3")


@gpu
@pytest.mark.parametrize("opt", ["sgd", "adam"])
@pytest.mark.parametrize("mode", ["legacy", "phased", "mcd"])
def test_stats_change_no_bit_of_the_step(opt, mode):
    """stats=True against stats=False on copies of one model over four steps (the last a short batch): the loss,
    every gradient and every updated parameter are bit-identical, and stats=True adds exactly one launch."""
    import copy

    from ta3n_b200.train import Adam, SGDNesterov, TrainStep
    model_a = _gpu_model(mcd=mode == "mcd")
    model_b = copy.deepcopy(model_a)
    mk = lambda: SGDNesterov(lr=0.05) if opt == "sgd" else Adam(lr=1e-3)      # noqa: E731
    kw = dict(beta=[0.75, 0.75, 0.5], mode="phased" if mode == "phased" else "legacy", mu=0.7 if mode == "mcd" else 0.0,
              seed=99)
    Bs, Bt, T = 8, 6, 5
    sa = TrainStep(model_a, Bs, Bt, optimizer=mk(), stats=True, **kw)
    sb = TrainStep(model_b, Bs, Bt, optimizer=mk(), **kw)
    assert sa.launches_per_step == sb.launches_per_step + 1
    g = torch.Generator().manual_seed(29)
    for i, (vs, vt) in enumerate(((Bs, Bt),) * 3 + ((5, 2),)):
        xs, xt = torch.randn(vs, T, 2048, generator=g), torch.randn(vt, T, 2048, generator=g)
        y = torch.randint(0, 7, (vs,), generator=g)
        la, lb = sa(xs, xt, y).clone(), sb(xs, xt, y).clone()
        torch.cuda.synchronize()
        assert torch.equal(la, lb), i
        assert torch.equal(sa.flat_grad, sb.flat_grad), i
        assert torch.equal(sa.flat_param, sb.flat_param), i
    assert sa.stats().steps == 4


@gpu
@pytest.mark.parametrize("use_graph", [True, False])
def test_reset_async_reads_and_replays(use_graph):
    """stats_async() agrees with stats(); reset_stats() starts a new epoch; the same batch replayed gives the same
    vals bit for bit; the warm-up of the capture is not counted."""
    from ta3n_b200.train import TrainStep
    model = _gpu_model()
    Bs, Bt, T = 8, 6, 5
    step = TrainStep(model, Bs, Bt, beta=[0.75, 0.75, 0.5], stats=True, use_graph=use_graph)
    assert step.stats().steps == 0 and step.stats().loss.count == 0
    g = torch.Generator().manual_seed(31)
    xs, xt = torch.randn(Bs, T, 2048, generator=g), torch.randn(Bt, T, 2048, generator=g)
    y = torch.randint(0, 7, (Bs,), generator=g)
    step(xs, xt, y)
    snap = step.stats_async()
    step(xs, xt, y)
    first = snap.result()
    st = step.stats()
    assert first.steps == 1 and st.steps == 2
    assert st.loss.val == first.loss.val and st.loss.sum == 2 * first.loss.sum
    for m in LOSS_METERS:
        assert getattr(st, m).val == getattr(first, m).val
    assert step.stats_async().result() == st
    step.reset_stats()
    empty = step.stats()
    assert empty.steps == 0 and all(getattr(empty, m).count == 0 for m in LOSS_METERS) and empty.rows == 0
    step(xs, xt, y)
    again = step.stats()
    assert again.steps == 1 and again.loss_c == first.loss_c and again.top1 == first.top1
    no_stats = TrainStep(_gpu_model(), Bs, Bt, beta=[0.75, 0.75, 0.5], use_graph=use_graph)
    with pytest.raises(ValueError, match="stats=True"):
        no_stats.stats()
    with pytest.raises(ValueError, match="stats_topk"):
        TrainStep(_gpu_model(), Bs, Bt, beta=[0.75, 0.75, 0.5], stats=True, stats_topk=(1, 8))


@gpu
def test_device_sampler_epochs_with_reset(tmp_path):
    """Two epochs from the device sampler with reset_stats() between them at fixed weights: the second epoch's
    meters equal the first's (same weights; the sampler reshuffles, and an epoch mean does not depend on the order
    beyond rounding) in counts, and its val is that of its own last batch."""
    from ta3n_b200 import dataset as D
    from ta3n_b200.train import TrainStep
    z, meta = _golden()
    case = "shipped"
    c = gen.CASES[case]
    model = _case_model(case, meta)
    xs, labels, xt, _, _ = gen.case_inputs(c)
    src, tgt = _shards(tmp_path, c, xs, labels, xt)
    sampler = D.DevicePairedSampler(D.DeviceFeatureBank(src), D.DeviceFeatureBank(tgt), (c["bs"], c["bt"]),
                                    seed=gen.SAMPLER_SEED)
    step = TrainStep(model, c["bs"], c["bt"], beta=list(gen.BETA), sampler=sampler, stats=True)
    epochs = []
    for _ in range(2):
        step.reset_stats()
        for _ in range(sampler.start_epoch()):
            step.run()
        epochs.append(step.stats())
    _check_epoch_against_fixture(epochs[0], z, case)
    for m in LOSS_METERS + ("top1", "top5"):
        assert getattr(epochs[1], m).count == getattr(epochs[0], m).count
    assert abs(epochs[1].loss_c.avg - epochs[0].loss_c.avg) <= 1e-6 * abs(epochs[0].loss_c.avg)
    assert epochs[1].correct == epochs[0].correct
