"""Validation in one CUDA graph: the validation head (ta3n_eval_head), the ordered device gather (ta3n_gather_rows),
DeviceEvalSampler and EvalStep.

CPU: the fp64 oracle of validate() (oracle/eval_oracle.py) against the reference's validate() (tests/golden/
eval_golden.npz), the C ABI's argument checks, what EvalStep refuses.
GPU: the head alone against fp64; EvalStep against the golden fixtures and against this repository's
VideoModel.forward(val, val, is_train=False); host batches against the device sampler; evaluation interleaved with
training.
"""
import copy
import json
import os
import types

import numpy as np
import pytest
import torch

from oracle import eval_oracle as eo
from oracle import gen_golden_eval as gen
from ta3n_b200 import dataset as D
from tests.golden_util import TOL_PATH, assert_close

gpu = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ENGINES = ["fp32", "tf32x3", "tf32"]


def _golden():
    z = np.load(os.path.join(HERE, "golden", "eval_golden.npz"))
    return z, json.loads(bytes(z["meta_json"]).decode())


def _shard(root, name, n, T, F, seed, num_dataload=None, n_class=5):
    """A packed shard as pack_list writes it (fp32 (n, T, F) .npy + .json with the labels)."""
    rng = np.random.default_rng(seed)
    path = os.path.join(str(root), name + ".npy")
    np.save(path, rng.standard_normal((n, T, F), dtype=np.float32))
    with open(path + ".json", "w") as f:
        json.dump({"num_segments": T, "labels": [int(v) for v in rng.integers(0, n_class, n)]}, f)
    return D.PackedTSNDataSet(path, num_dataload=num_dataload)


# ------------------------------------------------------------------------------------------------
# CPU: the oracle against the reference's validate()
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(gen.CASES))
def test_oracle_reproduces_reference_validate(case):
    """Per-batch loss, prec@1 / prec@5 (as counts) and the epoch averages of the reference's validate() from the
    fp64 oracle on the reference's logits; the confusion counts add up to the rows and their diagonal to prec@1."""
    z, _ = _golden()
    c, k = gen.CASES[case], case + "/"
    w = z[k + "class_weight"] if k + "class_weight" in z.files else None
    res = eo.epoch_metrics(z[k + "logits"], z[k + "labels"], c["batch"], w, topk=(1, 5))
    ref = z[k + "batch"]
    assert len(res["batches"]) == ref.shape[0] == -(-c["N"] // c["batch"])
    for b, (loss, p1, p5, n) in zip(res["batches"], ref):
        assert b["n"] == n
        assert abs(b["loss"] - loss) <= 1e-5 * abs(loss)                  # the reference computes in fp32
        assert b["correct"] == (round(p1 * n / 100), round(p5 * n / 100))
    loss, p1, p5 = z[k + "epoch"]
    assert abs(res["loss"] - loss) <= 1e-5 * abs(loss)
    assert abs(res["prec"][0] - p1) <= 1e-4 and abs(res["prec"][1] - p5) <= 1e-4
    assert res["confusion"].sum() == c["N"] and np.trace(res["confusion"]) == res["correct"][0]


def test_oracle_tie_rule():
    """Ties rank by class index: the label beats equal logits of higher classes and loses to lower ones."""
    z = np.array([[1.0, 3.0, 3.0, 0.0, 3.0], [2.0, 2.0, 2.0, 2.0, 2.0]])
    assert eo.label_rank(z, np.array([2, 0])).tolist() == [1, 0]
    assert eo.label_rank(z, np.array([4, 4])).tolist() == [2, 4]
    assert eo.top1(z).tolist() == [1, 0]
    m = eo.batch_metrics(z, np.array([1, 3]), topk=(1, 4))
    assert m["correct"] == (1, 2)
    # a NaN logit anywhere in a row: NaN loss, a hit at no k, no confusion cell; a row of -inf: every class ties
    zn = np.array([[np.nan, 1.0, 0.0], [0.0, np.nan, 1.0], [-np.inf, -np.inf, -np.inf], [0.0, 2.0, 1.0]])
    yn = np.array([0, 2, 1, 1])
    assert eo.label_rank(zn, yn).tolist() == [eo.UNRANKED, eo.UNRANKED, 1, 0]
    res = eo.epoch_metrics(zn, yn, 4, topk=(1, 2))
    assert np.isnan(res["loss"]) and res["correct"] == (1, 2)
    assert res["confusion"].sum() == 2 and res["confusion"][1, 0] == 1 and res["confusion"][1, 1] == 1


# ------------------------------------------------------------------------------------------------
# CPU: argument checks of the C ABI, refusals of EvalStep
# ------------------------------------------------------------------------------------------------
def test_eval_head_validates_arguments_without_gpu():
    import ctypes

    from ta3n_b200 import _lib
    lib = _lib.load()
    ks = (ctypes.c_int * 3)(1, 5, 12)
    names = ["feat", "rows", "H", "C", "Wc", "bc", "labels", "cw", "valid", "n_k", "k", "attn", "R", "attn_ld",
             "logits", "accum", "conf", "scores", "attn_out", "n_epoch", "ws", "ws_bytes", "stream"]
    ok = [256, 64, 256, 12, 512, 768, 1024, None, 1280, 3, ks, None, 4, 4, 1536, 1792, 2048, None, None, 0, 2304,
          lib.ta3n_eval_workspace_bytes(64), None]

    def call(**kw):
        args = dict(zip(names, ok))
        args.update(kw)
        return lib.ta3n_eval_head(*[args[n] for n in names])

    for kw, msg in ((dict(rows=0), b"rows, H and C"), (dict(C=0), b"rows, H and C"), (dict(n_k=0), b"top-k"),
                    (dict(n_k=5), b"top-k"), (dict(k=None), b"top-k"),
                    (dict(C=4), b"outside [1, C=4]"), (dict(k=(ctypes.c_int * 3)(0, 1, 2)), b"outside"),
                    (dict(feat=None), b"null pointer"), (dict(labels=None), b"null pointer"),
                    (dict(valid=None), b"null pointer"), (dict(accum=None), b"null pointer"),
                    (dict(accum=1796), b"8-byte aligned"), (dict(conf=2052), b"8-byte aligned"),
                    (dict(scores=4096), b"n_epoch"), (dict(attn_out=4096, n_epoch=10), b"attn_out"),
                    (dict(attn_out=4096, n_epoch=10, attn=512, attn_ld=3), b"attn_out"),
                    (dict(ws=None), b"workspace"), (dict(ws=2308), b"workspace")):
        assert call(**kw) == 1, kw
        err = lib.ta3n_last_error()
        assert b"ta3n_eval_head" in err and msg in err, (kw, err)
    assert call(ws_bytes=8) == 2 and b"workspace too small" in lib.ta3n_last_error()
    assert call(H=4096) == 4 and b"too wide" in lib.ta3n_last_error()
    assert lib.ta3n_eval_workspace_bytes(0) == 0 and lib.ta3n_eval_workspace_bytes(9) >= 2 * 64


def test_gather_rows_validates_arguments_without_gpu():
    from ta3n_b200 import _lib
    lib = _lib.load()
    names = ["bank", "n_rows", "rows", "labels", "n_epoch", "batch", "x", "y", "row_floats", "valid", "state", "stream"]
    ok = [256, 10, 512, 768, 10, 4, 1024, 1280, 40, 2304, 2560, None]

    def call(**kw):
        args = dict(zip(names, ok))
        args.update(kw)
        return lib.ta3n_gather_rows(*[args[n] for n in names])

    for kw, msg in ((dict(bank=None), b"null pointer"), (dict(labels=None), b"null pointer"),
                    (dict(y=None), b"null pointer"), (dict(valid=None), b"null valid_rows"),
                    (dict(state=None), b"null valid_rows"), (dict(batch=0), b"batch"), (dict(batch=70000), b"batch"),
                    (dict(row_floats=42), b"multiple of 4"), (dict(n_epoch=0), b"empty epoch"),
                    (dict(n_rows=1 << 31), b"2^31"), (dict(bank=260), b"16-byte aligned"),
                    (dict(x=1028), b"16-byte aligned"), (dict(n_rows=1 << 30, row_floats=1 << 40), b"too large")):
        assert call(**kw) == 1, kw
        err = lib.ta3n_last_error()
        assert b"ta3n_gather_rows" in err and msg in err, (kw, err)


def _cpu_model(**kw):
    from ta3n_b200.models import VideoModel
    args = dict(train_segments=5, val_segments=5, fc_dim=64, verbose=False)
    args.update(kw)
    return VideoModel(5, "video", "trn-m", "RGB", **args)


def test_eval_step_refuses_several_ranks_and_a_cpu_model(monkeypatch):
    from ta3n_b200 import Ta3nError
    from ta3n_b200 import evaluate
    with pytest.raises(Ta3nError, match="CUDA device"):
        evaluate.EvalStep(_cpu_model(), 8)
    monkeypatch.setattr(evaluate.dist, "is_initialized", lambda: True)
    monkeypatch.setattr(evaluate.dist, "get_world_size", lambda group=None: 2)
    with pytest.raises(NotImplementedError, match="single rank"):
        evaluate.EvalStep(_cpu_model(), 8)


def test_eval_result_precisions():
    from ta3n_b200.evaluate import EvalResult
    r = EvalResult(loss=1.0, n=8, topk=(1, 5), correct=(2, 6), confusion=np.zeros((5, 5)), batches=1)
    assert (r.prec1, r.prec5, r.prec(5)) == (25.0, 75.0, 75.0)


# ------------------------------------------------------------------------------------------------
# GPU: the head alone against fp64
# ------------------------------------------------------------------------------------------------
def _head_call(lib, feat, W, b, labels, cw, valid, ks, logits, acc, conf, scores=None, n_epoch=0, attn=None,
               attn_out=None, ws=None):
    import ctypes
    rows, H = feat.shape
    C = W.shape[0]
    R = 0 if attn is None else attn.shape[1]
    karr = (ctypes.c_int * len(ks))(*ks)
    p = lambda t: None if t is None else t.data_ptr()    # noqa: E731
    return lib.ta3n_eval_head(p(feat), rows, H, C, p(W), p(b), p(labels), p(cw), p(valid), len(ks), karr, p(attn), R,
                              R, p(logits), p(acc), p(conf), p(scores), p(attn_out), n_epoch, p(ws), ws.numel(),
                              torch.cuda.current_stream().cuda_stream)


def _read_acc(acc, n_k):
    h = acc.cpu().numpy()
    return dict(loss_sum=float(h[0:1].view(np.float64)[0]), n=int(h[1]), correct=tuple(int(v) for v in h[2:2 + n_k]),
                batch=int(h[6:7].view(np.int32)[0]), arrive=int(h[6:7].view(np.int32)[1]))


@gpu
@pytest.mark.parametrize("C", [5, 12, 30, 1000, 1500])
@pytest.mark.parametrize("weighted", [False, True])
def test_eval_head_against_fp64(C, weighted):
    """Several batches (the last one short, padding rows garbage) through ONE captured graph replayed per batch, with
    exact ties planted (duplicated classifier rows): logits within 2e-6 normwise of fp64, counts and confusion exact
    under the documented tie rule, the epoch loss within 1e-6, scores / attention in dataset order, and a second
    epoch bit-identical to the first.  C = 1000 / 1500 stream the classifier through shared memory."""
    from ta3n_b200 import _lib
    lib = _lib.load()
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(C + weighted)
    rows, H, R, N = 24, 256, 4, 61          # 3 batches: 24 + 24 + 13
    W = torch.randn(C, H, generator=g) * 0.1
    b = torch.randn(C, generator=g) * 0.1
    W[C - 1], b[C - 1] = W[1], b[1]         # class C-1 ties class 1 on every row
    W[3], b[3] = W[2], b[2]                 # class 3 ties class 2
    X = torch.randn(N, H, generator=g)
    Y = torch.randint(0, C, (N,), generator=g)
    Y[::5] = C - 1                          # labels on the tied classes: ranked after / before their twins
    Y[1::7] = 1
    Y[2::9] = 2
    A = torch.randn(N, R, generator=g)
    cw = (0.5 + torch.rand(C, generator=g)) if weighted else None
    ks = (1, 5, C)
    feat = torch.zeros(rows, H, device=dev)
    lab = torch.zeros(rows, device=dev, dtype=torch.int64)
    attn = torch.zeros(rows, R, device=dev)
    valid = torch.zeros(1, device=dev, dtype=torch.int32)
    Wd, bd = W.to(dev), b.to(dev)
    cwd = None if cw is None else cw.to(dev)
    logits = torch.zeros(rows, C, device=dev)
    acc = torch.zeros(8, device=dev, dtype=torch.int64)
    conf = torch.zeros(C, C, device=dev, dtype=torch.int64)
    scores = torch.full((N, C), float("nan"), device=dev)
    attn_out = torch.full((N, R), float("nan"), device=dev)
    ws = torch.zeros(lib.ta3n_eval_workspace_bytes(rows), device=dev, dtype=torch.uint8)
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        _lib.check(_head_call(lib, feat, Wd, bd, lab, cwd, valid, ks, logits, acc, conf, scores, N, attn, attn_out,
                              ws))

    def epoch():
        acc.zero_(), conf.zero_()
        got = []
        for a in range(0, N, rows):
            n = min(rows, N - a)
            feat.normal_(), lab.random_(0, C), attn.normal_()       # padding rows: whatever is left there
            feat[:n].copy_(X[a:a + n]), lab[:n].copy_(Y[a:a + n]), attn[:n].copy_(A[a:a + n])
            valid.fill_(n)
            gr.replay()
            got.append(logits[:n].clone())
        torch.cuda.synchronize()
        return torch.cat(got), _read_acc(acc, len(ks)), conf.cpu().numpy(), scores.clone(), attn_out.clone()

    z, st, cf, sc, ao = epoch()
    z64 = X.double() @ W.double().t() + b.double()
    assert (z.double().cpu() - z64).norm() <= 2e-6 * z64.norm()
    zc = z.double().cpu().numpy()
    assert np.all(zc[:, C - 1] == zc[:, 1]) and np.all(zc[:, 3] == zc[:, 2])     # the ties are exact
    ref = eo.epoch_metrics(zc, Y.numpy(), rows, None if cw is None else cw.numpy(), topk=ks)
    assert st["n"] == N and st["batch"] == 3 and st["arrive"] == 0
    assert st["correct"] == ref["correct"]
    assert np.array_equal(cf, ref["confusion"])
    assert abs(st["loss_sum"] / N - ref["loss"]) <= 1e-6 * abs(ref["loss"])
    ref64 = eo.epoch_metrics(z64.numpy(), Y.numpy(), rows, None if cw is None else cw.numpy(), topk=ks)
    assert abs(st["loss_sum"] / N - ref64["loss"]) <= 1e-5 * abs(ref64["loss"])
    assert torch.equal(sc.cpu(), z.cpu()) and torch.equal(ao.cpu(), A)
    z2, st2, cf2, sc2, ao2 = epoch()
    assert torch.equal(z2, z) and st2 == st and np.array_equal(cf2, cf) and torch.equal(sc2, sc)


@gpu
@pytest.mark.parametrize("C", [7, 40, 1000])
def test_eval_head_rows_with_nan_or_inf_logits(C):
    """Rows whose logits are all NaN (a NaN feature row, real and padding), rows with one NaN logit (a NaN bias entry,
    the label's own logit among them) and rows of -inf logits (a -inf bias): the confusion counts stay inside their
    [C, C] buffer (sentinels on both sides untouched), NaN rows are hits at no k and count in no cell, -inf rows rank by
    the tie rule, every count equals the fp64 oracle's, the loss is NaN, and the accumulator advances normally."""
    from ta3n_b200 import _lib
    lib = _lib.load()
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(C)
    rows, H, n = 16, 32, 13
    ks = (1, 5)
    W = (torch.randn(C, H, generator=g) * 0.3).to(dev)
    acc = torch.zeros(8, device=dev, dtype=torch.int64)
    pad = 1024
    conf_buf = torch.full((2 * pad + C * C,), -7, device=dev, dtype=torch.int64)
    conf = conf_buf[pad:pad + C * C].view(C, C)
    ws = torch.zeros(lib.ta3n_eval_workspace_bytes(rows), device=dev, dtype=torch.uint8)
    valid = torch.full((1,), n, device=dev, dtype=torch.int32)
    logits = torch.zeros(rows, C, device=dev)
    conf.zero_()
    got, labs = [], []
    for case in ("nan_rows", "nan_column", "minus_inf"):
        feat = torch.randn(rows, H, generator=g)
        lab = torch.randint(0, C, (rows,), generator=g)
        b = torch.randn(C, generator=g) * 0.1
        if case == "nan_rows":
            feat[3] = float("nan")                   # a real row
            feat[14] = float("nan")                  # a padding row
        elif case == "nan_column":
            b[2] = float("nan")                      # every row has a NaN logit; some have it as their label's
            lab[:4] = 2
        else:
            b[:] = float("-inf")
        _lib.check(_head_call(lib, feat.to(dev), W, b.to(dev), lab.to(dev), None, valid, ks, logits, acc, conf,
                              ws=ws))
        torch.cuda.synchronize()
        got.append(logits[:n].double().cpu().numpy())
        labs.append(lab[:n].numpy())
    st = _read_acc(acc, len(ks))
    assert torch.all(conf_buf[:pad] == -7) and torch.all(conf_buf[pad + C * C:] == -7)
    z, y = np.concatenate(got), np.concatenate(labs)
    assert np.isnan(z[3]).all() and np.isnan(z[n:2 * n, 2]).all() and np.isneginf(z[2 * n:]).all()
    ref = eo.epoch_metrics(z, y, n, topk=ks)
    assert st["n"] == 3 * n and st["batch"] == 3 and st["arrive"] == 0
    assert st["correct"] == ref["correct"]
    assert np.array_equal(conf.cpu().numpy(), ref["confusion"])
    assert conf.sum().item() == n - 1 + n            # first batch less its NaN row, the -inf batch whole
    assert np.isnan(st["loss_sum"])


# ------------------------------------------------------------------------------------------------
# GPU: EvalStep
# ------------------------------------------------------------------------------------------------
def _case_model(case, meta):
    from ta3n_b200.models import VideoModel
    c = gen.CASES[case]
    params = gen.case_params(c, meta[case + "/param_order"])
    m = VideoModel(c["C"], "video", c["agg"], "RGB", train_segments=c["T"], val_segments=c["Tv"], fc_dim=c["F"],
                   use_attn=c["use_attn"], use_attn_frame=c["attn_frame"], ens_DA=c["ens"], verbose=False)
    m.load_state_dict(params)                      # strict: every key of the reference's state_dict, nothing else
    return m.cuda().eval()


def _margin_flips(got_correct_rows, ref_correct_rows, z64, labels, k):
    """Rows whose top-k correctness differs, and how many of them lie within the rounding margin."""
    diff = got_correct_rows != ref_correct_rows
    margin = eo.topk_margin(z64, labels, k)
    near = margin < 1e-4 * np.abs(z64).max()
    return int(diff.sum()), int((diff & ~near).sum())


@gpu
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case", list(gen.CASES))
def test_eval_step_against_reference_validate(case, engine):
    """EvalStep fed the golden inputs as host batches (short last batch) against the reference's validate(): logits
    and attention within TOL_PATH (+ the reference's own fp32 noise), epoch loss within 1e-4, top-k correctness equal
    except on rows within the rounding margin."""
    import ta3n_b200
    from ta3n_b200.evaluate import EvalStep
    ta3n_b200.set_gemm_engine(engine)
    z, meta = _golden()
    c, k = gen.CASES[case], case + "/"
    model = _case_model(case, meta)
    x, labels, weight = gen.case_inputs(c)
    ev = EvalStep(model, c["batch"], class_weight=weight, topk=(1, 5), keep_scores=True, epoch_rows=c["N"])
    ev.reset()
    for a in range(0, c["N"], c["batch"]):
        ev(x[a:a + c["batch"]], labels[a:a + c["batch"]])
    res = ev.result()
    assert res.n == c["N"] and res.batches == -(-c["N"] // c["batch"])
    assert_close(res.scores, z[k + "logits"], TOL_PATH, f"{case} logits", noise=float(z[k + "noise/logits"]))
    assert_close(res.attn, z[k + "attn"], TOL_PATH, f"{case} attn", noise=float(z[k + "noise/attn"]))
    assert abs(res.loss - z[k + "epoch"][0]) <= 1e-4 * abs(z[k + "epoch"][0])
    ref = eo.epoch_metrics(z[k + "logits"], labels.numpy(), c["batch"], weight, topk=(1, 5))
    for i, kk in enumerate((1, 5)):
        got_rows = eo.label_rank(res.scores.double().cpu().numpy(), labels.numpy()) < kk
        ref_rows = eo.label_rank(z[k + "logits"], labels.numpy()) < kk
        n_diff, n_far = _margin_flips(got_rows, ref_rows, z[k + "logits"], labels.numpy(), kk)
        assert n_far == 0, (case, kk, n_diff)
        assert abs(res.correct[i] - ref["correct"][i]) <= n_diff
    assert model.training is False


@gpu
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case", ["transattn_T5_w", "general", "attnframe_T4", "avgpool_Tv7", "mcd"])
def test_eval_step_against_video_model_forward(case, engine):
    """EvalStep against this repository's VideoModel.forward(val, val, [0]*3, 0, is_train=False) on the same engine:
    the target half, scored by the fp64 oracle.  The model stays in train mode (EvalStep neither reads nor changes
    it: no dropout either way) and no .grad appears."""
    import ta3n_b200
    from ta3n_b200.evaluate import EvalStep
    ta3n_b200.set_gemm_engine(engine)
    z, meta = _golden()
    c = gen.CASES[case]
    model = _case_model(case, meta).train()
    x, labels, weight = gen.case_inputs(c)
    B = c["batch"]
    ev = EvalStep(model, B, class_weight=weight, keep_scores=True, epoch_rows=c["N"])
    ev.reset()
    for a in range(0, c["N"], B):
        ev(x[a:a + B], labels[a:a + B])
    res = ev.result()
    assert model.training is True
    assert all(p.grad is None for p in model.parameters())
    model.eval()
    outs, attns = [], []
    with torch.no_grad():
        for a in range(0, c["N"], B):
            xb = x[a:a + B].cuda()
            o = model(xb, xb, [0] * 3, 0, is_train=False, reverse=False)
            outs.append(o[6])
            attns.append(o[5].reshape(xb.shape[0], -1))
    ref_z, ref_a = torch.cat(outs).double().cpu(), torch.cat(attns).double().cpu()
    assert_close(res.scores, ref_z, 2e-5 if engine != "tf32" else TOL_PATH, f"{case} logits", noise=1e-7)
    assert_close(res.attn, ref_a, 2e-5 if engine != "tf32" else TOL_PATH, f"{case} attn", noise=1e-7)
    ref = eo.epoch_metrics(ref_z.numpy(), labels.numpy(), B, weight, topk=(1, 5))
    assert abs(res.loss - ref["loss"]) <= 1e-4 * abs(ref["loss"])
    for i, kk in enumerate((1, 5)):
        got_rows = eo.label_rank(res.scores.double().cpu().numpy(), labels.numpy()) < kk
        ref_rows = eo.label_rank(ref_z.numpy(), labels.numpy()) < kk
        n_diff, n_far = _margin_flips(got_rows, ref_rows, ref_z.numpy(), labels.numpy(), kk)
        assert n_far == 0 and abs(res.correct[i] - ref["correct"][i]) <= n_diff


@gpu
@pytest.mark.parametrize("agg", ["trn-m", "avgpool"])
def test_host_batches_equal_device_sampler(tmp_path, agg):
    """The same epoch through host batches (ev(data, label)) and through DeviceEvalSampler: bit-identical logits,
    attention, accumulator and confusion, with a short last batch and num_dataload tiling; twice, to check the
    sampler's rewind and the accumulator's reset."""
    from ta3n_b200.evaluate import EvalStep
    from ta3n_b200.models import VideoModel
    T, B = 5, 8
    ds = _shard(tmp_path, "v", 17, T, 2048, 5, num_dataload=29, n_class=6)          # 29 positions: 8+8+8+5
    torch.manual_seed(0)
    model = VideoModel(6, "video", agg, "RGB", train_segments=5, val_segments=T, fc_dim=128, verbose=False).cuda()
    sampler = D.DeviceEvalSampler(D.DeviceFeatureBank(ds), B)
    assert len(sampler) == 4
    ev_dev = EvalStep(model, B, sampler=sampler, keep_scores=True)
    ev_host = EvalStep(model, B, keep_scores=True, epoch_rows=len(ds))
    assert ev_dev.launches_per_batch == 0          # not captured before the first epoch
    for _ in range(2):
        r_dev = ev_dev.run_epoch()
        ev_host.reset()
        for a in range(0, len(ds), B):
            idx = np.arange(a, min(a + B, len(ds)))
            ev_host(torch.from_numpy(np.stack([ds[int(i)][0].numpy() for i in idx])), torch.from_numpy(ds.labels[idx]))
        r_host = ev_host.result()
        assert ev_dev.launches_per_batch == ev_host.launches_per_batch + 1
        assert r_dev.n == r_host.n == 29 and r_dev.batches == r_host.batches == 4
        assert r_dev.loss == r_host.loss and r_dev.correct == r_host.correct
        assert np.array_equal(r_dev.confusion, r_host.confusion)
        assert torch.equal(r_dev.scores, r_host.scores) and torch.equal(r_dev.attn, r_host.attn)
        assert ev_dev.valid.item() == 5
    with pytest.raises(RuntimeError, match="device sampler"):
        ev_dev(torch.zeros(2, T, 2048), torch.zeros(2, dtype=torch.int64))
    sampler.start_epoch()
    for _ in range(4):
        sampler.take()
    with pytest.raises(RuntimeError, match="all have run"):
        sampler.take()


@gpu
def test_interleaved_training_is_unchanged_and_evaluation_sees_current_weights(tmp_path):
    """Train an epoch (TrainStep + DevicePairedSampler), validate, train another: the training trajectory (loss,
    parameters, momentum after every step) is bit-identical to the run without validation, and each validation equals
    a freshly built EvalStep's on the weights of that moment -- although this EvalStep was built BEFORE the TrainStep
    flattened the parameters (re-capture)."""
    from ta3n_b200.evaluate import EvalStep
    from ta3n_b200.models import VideoModel
    from ta3n_b200.train import SGDNesterov, TrainStep
    T, batch = 5, (8, 6)
    src, tgt, val = (_shard(tmp_path, "s", 21, T, 2048, 1), _shard(tmp_path, "t", 14, T, 2048, 2),
                     _shard(tmp_path, "v", 19, T, 2048, 3))
    banks = [D.DeviceFeatureBank(s) for s in (src, tgt, val)]
    torch.manual_seed(0)
    model_a = VideoModel(5, "video", "trn-m", "RGB", train_segments=5, val_segments=5, fc_dim=96,
                         verbose=False).cuda().train()
    model_b = copy.deepcopy(model_a)
    ev = EvalStep(model_a, 8, sampler=D.DeviceEvalSampler(banks[2], 8))
    first = ev.run_epoch()
    kw = dict(beta=[0.75, 0.75, 0.5], seed=9)
    sa, sb = D.DevicePairedSampler(banks[0], banks[1], batch, seed=4), D.DevicePairedSampler(banks[0], banks[1],
                                                                                            batch, seed=4)
    step_a = TrainStep(model_a, *batch, sampler=sa, optimizer=SGDNesterov(lr=0.05), **kw)
    step_b = TrainStep(model_b, *batch, sampler=sb, optimizer=SGDNesterov(lr=0.05), **kw)
    results = [first]
    for epoch in range(2):
        assert sa.start_epoch() == sb.start_epoch()
        for _ in range(sa.n_iter):
            la, lb = step_a.run().clone(), step_b.run().clone()
            torch.cuda.synchronize()
            assert torch.equal(la, lb)
            assert torch.equal(step_a.flat_param, step_b.flat_param)
            assert torch.equal(step_a.momentum_buf, step_b.momentum_buf)
        res = ev.run_epoch()
        fresh = EvalStep(model_a, 8, sampler=D.DeviceEvalSampler(banks[2], 8)).run_epoch()
        assert res.loss == fresh.loss and res.correct == fresh.correct
        assert np.array_equal(res.confusion, fresh.confusion)
        results.append(res)
    assert results[0].loss != results[1].loss != results[2].loss      # the weights moved between validations
    assert step_a.step_counter.item() == step_b.step_counter.item()
