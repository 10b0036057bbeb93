"""The precise tensor-core kernel (tf32x3): fp32-grade results against fp64, in every operand layout it runs.

  K-major x K-major (the forward layers, seg_gemm_tc_x3_kernel<true, true>): through ta3n_gemm_tn, one case per
                     schedule regime of the persistent kernel (listed LPT tasks, several tasks per CTA and so reuse of
                     the two context slots, the strided order beyond 1024 tasks, split K with the vectorised and the
                     scalar reduce, M = 1, ragged slabs and tiles), and through the operator entry points whose
                     epilogues and multi-group plans the model runs (shared layer with both dropouts, the forward
                     batch of the frame discriminator and the TRN cut into two launches, the relation
                     discriminators on a strided A, 'general' attention on the generic epilogue).
  M-major x N-major (weight gradients of the 256 x 256 discriminator layers): through ta3n_gemm_ex, whose small
                     M-major x N-major products run on the precise kernel under tf32x3.
  K-major x N-major (data gradients with TA3N_X3_DGRAD=1): through ta3n_disc_bwd in a child process, because the
                     library reads that variable once.

A plain tf32 product is ~3e-4 off normwise; the bound below is 15x tighter.  The forward cases also hold every 128 x 128
output tile to it (relative to the tile, or to the tensor's RMS tile norm where the tile is small), so one wrong task
cannot hide in the norm of the rest; they pre-fill outputs with NaN behind a guard region that must stay untouched,
name the kernels that ran (torch.profiler) and assert the schedule regime they cover through the planner's C ABI.
"""
import ctypes as C
import json
import math
import os
import re
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
X3_TOL = 2e-5
ROW_TOL = 2e-4           # the row kernels after the GEMMs (relation heads, attention, pooling): fp32 FMA chains
TILE = 128               # output tile of the tensor-core kernels
MAX_LISTED = 1024        # tasks a launch can list (kX3MaxTasks); beyond: strided order
MAX_CTAS = 144           # kX3MaxCtas
MAX_SEGS = 128           # segments one launch holds (kMaxSegs)
SCRATCH_BYTES = 48 << 20
GUARD = 4096             # floats (16 KB) behind every output
SENTINEL = -1234.5
SEED = 0xC0FFEE1234567891


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm()).item()


def _dev():
    return torch.device("cuda:0")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


class _Out:
    """An fp32 output pre-filled with NaN, followed by GUARD floats of SENTINEL that the kernels must not touch."""

    def __init__(self, *shape):
        self.n = math.prod(shape)
        self.buf = torch.full((self.n + GUARD,), float("nan"), device=_dev())
        self.buf[self.n:] = SENTINEL
        self.t = self.buf[:self.n].view(*shape)

    def ptr(self):
        return self.t.data_ptr()

    def check_guard(self, what):
        bad = (self.buf[self.n:] != SENTINEL).sum().item()
        assert bad == 0, f"{what}: {bad} guard floats behind the output were written"


def _mm(a, b):
    """a @ b.T in fp64 (returned on the CPU): computed on the GPU from 1 GFLOP on, else on the CPU."""
    big = 2.0 * a.shape[0] * b.shape[0] * a.shape[1] >= 1e9
    d = _dev() if big else torch.device("cpu")
    return (a.to(d, torch.float64) @ b.to(d, torch.float64).t()).cpu()


def _check_tiles(what, got, ref, tol=X3_TOL):
    """got (fp32) against ref (fp64), both [..., M, N] (a stack of GEMM outputs): normwise and per 128 x 128 tile,
    ||C_t - R_t|| <= tol * max(||R_t||, ||R|| / sqrt(tiles)).  Returns the worst tile's err / bound."""
    dev = _dev()
    ref = ref.to(dev, torch.float64)
    got = got.detach().to(dev, torch.float64)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert torch.isfinite(got).all(), f"{what}: non-finite values (an output element was not written)"
    M, N = ref.shape[-2], ref.shape[-1]
    got, ref = got.reshape(-1, M, N), ref.reshape(-1, M, N)
    pm, pn = -M % TILE, -N % TILE
    tm, tn = (M + pm) // TILE, (N + pn) // TILE

    def tiles(x):
        x = torch.nn.functional.pad(x, (0, pn, 0, pm))
        return x.reshape(x.shape[0], tm, TILE, tn, TILE).pow(2).sum((2, 4)).sqrt()

    diff = got - ref
    total = ref.norm().item()
    err = diff.norm().item() / total
    assert err < tol, f"{what}: normwise rel err {err:.2e} (bound {tol:.0e})"
    e, r = tiles(diff), tiles(ref)
    bound = tol * torch.clamp(r, min=total / math.sqrt(e.numel()))
    ratio = e / bound
    worst = ratio.max().item()
    idx = [int(i) for i in torch.nonzero(ratio == ratio.max())[0]]
    assert worst <= 1.0, f"{what}: tile (plane, row, col) {idx} err {e.flatten()[ratio.argmax()].item():.3e} is " \
                         f"{worst:.2f}x its bound (normwise {err:.2e})"
    headroom = f"{1 / worst:.1f}x headroom" if worst > 0 else "exact"
    print(f"[x3] {what}: normwise {err:.2e}, worst tile {worst:.3f} of its bound ({headroom})")
    return worst


def _kernels(fn, sessions=5):
    """Run fn under torch.profiler; the names of the CUDA kernels it launched, spaces removed.

    A profiler session now and then delivers no CUDA activity at all -- not even the probe kernel launched before fn.
    Such a session says nothing about fn, so fn (every caller's fn is idempotent) runs again under a fresh one, at most
    `sessions` times in all."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(sessions):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.ones(1, device=_dev()).add_(1)        # the session is recording before fn launches anything
            torch.cuda.synchronize()
            fn()
            torch.cuda.synchronize()
        names = [e.name.replace(" ", "") for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        names = [n for n in names if "memset" not in n.lower() and "memcpy" not in n.lower()]
        if names:
            return names
        print("[x3] the profiler session recorded no CUDA activity; running fn again under a fresh session")
    raise AssertionError(f"the profiler recorded no kernels in {sessions} sessions")


def _assert_kernels(names, x3_launches, reduce):
    """x3_launches of seg_gemm_tc_x3_kernel<true, true>, no other GEMM kernel; reduce in {None, 'v4', 'scalar'}."""
    x3 = [n for n in names if "seg_gemm_tc_x3_kernel<true,true>" in n]
    other = [n for n in names if ("seg_gemm" in n and n not in x3)]
    assert len(x3) == x3_launches, f"{len(x3)} precise K-major launches, expected {x3_launches}: {names}"
    assert not other, f"GEMM kernels other than the precise K-major one ran: {other}"
    v4 = sum("splitk_reduce_v4_kernel" in n for n in names)
    scalar = sum(re.search(r"splitk_reduce_kernel\b", n) is not None for n in names)
    if reduce == "v4":
        assert v4 >= 1 and scalar == 0, f"expected the vectorised split-K reduce: {names}"
    elif reduce == "scalar":
        assert scalar >= 1 and v4 == 0, f"expected the scalar split-K reduce: {names}"
    else:
        assert v4 == 0 and scalar == 0, f"unexpected split-K reduce: {names}"


class _Scratch:
    """Forward scratch registered for the block (the balanced planner may then split K), cleared afterwards."""

    def __init__(self, on):
        self.on = on
        self.buf = torch.empty(SCRATCH_BYTES, dtype=torch.uint8, device=_dev()) if on else None

    def __enter__(self):
        from ta3n_b200 import _lib
        if self.on:
            _lib.check(_lib.load().ta3n_set_forward_scratch(self.buf.data_ptr(), self.buf.numel()))
        return self

    def __exit__(self, *exc):
        from ta3n_b200 import _lib
        _lib.check(_lib.load().ta3n_set_forward_scratch(None, 0))
        return False


def _regime(shapes, scratch):
    """(split factors, tasks, tasks per CTA) of one precise launch of single-segment GEMMs [(M, N, K)] on this GPU."""
    from ta3n_b200 import _lib
    ks = _lib.plan_forward_splits(shapes, sms=_sms(), scratch_bytes=SCRATCH_BYTES)[0] if scratch else [1] * len(shapes)
    tasks = sum(math.ceil(M / TILE) * math.ceil(N / TILE) * k for (M, N, _), k in zip(shapes, ks))
    return ks, tasks, math.ceil(tasks / min(_sms(), MAX_CTAS))


def _reduce_kind(ks, vec_ok):
    return None if max(ks) == 1 else ("v4" if vec_ok and max(ks) <= 8 else "scalar")


def _run_twice(run, outs):
    """run() under the profiler, then again: every output bit-identical.  Returns the kernel names of the first run."""
    names = _kernels(run)
    for o in outs:
        assert torch.isfinite(o.t).all(), "an output element was not written"
    first = [o.t.clone() for o in outs]
    for o in outs:
        o.t.fill_(float("nan"))
    run()
    torch.cuda.synchronize()
    for a, o in zip(first, outs):
        assert torch.equal(a, o.t), "a second run gave a different result"
    return names


@pytest.fixture(autouse=True)
def _x3_engine():
    import ta3n_b200
    ta3n_b200.set_gemm_engine("tf32x3")
    yield


# ------------------------------------------------------------------------------------------------
# ta3n_gemm_tn: C = A B^T, both K-major -- one case per schedule regime
# ------------------------------------------------------------------------------------------------
# (M, N, K, scratch, expected split factor, tasks, tasks per CTA on 132 SMs, what it covers)
GEMM_TN = [
    (5, 4096, 8, False, 1, 32, 1, "K below one slab"),
    (300, 200, 36, False, 1, 6, 1, "ragged slab, ragged M and N"),
    (2560, 512, 2048, True, 3, 240, 2, "the cfg2 shared-layer shape, vectorised reduce"),
    (2000, 1100, 2044, False, 1, 144, 2, "run-ahead into the second slot, ragged K"),
    (2000, 1100, 2044, True, 2, 288, 3, "a slot reused with its barrier parity flipped"),
    (4096, 2560, 72, False, 1, 640, 5, "slot barriers over several phases, 3 slabs"),
    (4224, 4096, 64, False, 1, 1056, 8, "the strided schedule beyond 1024 tasks"),
    (1, 4096, 2048, True, 4, 128, 1, "M = 1, split partial planes"),
    (600, 300, 4100, True, 8, 120, 1, "uneven splits of 129 slabs"),
    (333, 257, 1000, True, 4, 36, 1, "odd N: scalar stores, scalar reduce"),
]


@pytest.mark.parametrize("M,N,K,scratch,ksplit,tasks,per_cta,covers", GEMM_TN,
                         ids=[f"{c[0]}x{c[1]}x{c[2]}-{'split' if c[3] else 'nosplit'}" for c in GEMM_TN])
def test_x3_gemm_tn_is_fp32_grade_in_every_regime(M, N, K, scratch, ksplit, tasks, per_cta, covers):
    from ta3n_b200 import _lib
    lib = _lib.load()
    if _sms() != 132:
        pytest.skip(f"the regimes are laid out for 132 SMs; this GPU has {_sms()}")
    ks, n_tasks, n_per_cta = _regime([(M, N, K)], scratch)
    assert (ks[0], n_tasks, n_per_cta) == (ksplit, tasks, per_cta), \
        f"planner moved the case out of its regime ({covers}): ksplit {ks[0]}, {n_tasks} tasks, {n_per_cta} per CTA"
    assert (n_tasks > MAX_LISTED) == ("strided" in covers)
    g = torch.Generator().manual_seed(M + 3 * N + 7 * K)
    A = torch.randn(M, K, generator=g)
    B = torch.randn(N, K, generator=g)
    ref = _mm(A, B)
    dA, dB = A.to(_dev()), B.to(_dev())
    out = _Out(M, N)
    st = torch.cuda.current_stream().cuda_stream
    run = lambda: _lib.check(lib.ta3n_gemm_tn(dA.data_ptr(), dB.data_ptr(), out.ptr(), M, N, K, st))  # noqa: E731
    with _Scratch(scratch):
        names = _run_twice(run, [out])
    _assert_kernels(names, 1, _reduce_kind(ks, N % 4 == 0))
    out.check_guard("gemm_tn")
    _check_tiles(f"gemm_tn {M}x{N}x{K} ksplit {ks[0]} ({covers})", out.t, ref)


def test_x3_split_k_with_strided_schedule():
    """Split K and more than 1024 tasks in one launch: one single-tile group with long K next to a 1024-tile group with
    short K.  The planner splits the long group 8 ways; the strided order then carries the partial planes and the
    vectorised reduce.  Through the forward batch (two frame-discriminator layers in one launch)."""
    from ta3n_b200 import _lib
    lib = _lib.load()
    if _sms() != 132:
        pytest.skip(f"the regime is laid out for 132 SMs; this GPU has {_sms()}")
    shapes = [(128, 128, 2048), (2048, 8192, 8)]
    ks, tasks, _ = _regime(shapes, True)
    assert ks == [8, 1] and tasks == 1032, (ks, tasks)
    g = torch.Generator().manual_seed(11)
    dev, st = _dev(), torch.cuda.current_stream().cuda_stream
    refs, outs, args = [], [], []
    for rows, Kh, K in shapes:
        x = torch.randn(rows, K, generator=g)
        W1 = torch.randn(Kh, K, generator=g) / K ** 0.5
        b1 = 0.1 * torch.randn(Kh, generator=g)
        W2 = torch.randn(2, Kh, generator=g) / Kh ** 0.5
        b2 = torch.randn(2, generator=g)
        refs.append(torch.relu(_mm(x, W1) + b1.double()))
        t = [v.to(dev) for v in (x, W1, b1, W2, b2)]
        hidden, logits = _Out(rows, Kh), _Out(rows, 2)
        outs += [hidden, logits]
        args.append((t, rows, K, Kh, hidden, logits))

    def run():
        _lib.check(lib.ta3n_fwd_batch_begin())
        for t, rows, K, Kh, hidden, logits in args:
            _lib.check(lib.ta3n_disc_fwd(t[0].data_ptr(), rows, K, Kh, t[1].data_ptr(), t[2].data_ptr(),
                                         t[3].data_ptr(), t[4].data_ptr(), hidden.ptr(), logits.ptr(), st))
        _lib.check(lib.ta3n_fwd_batch_flush(None, 0, st))

    with _Scratch(True):
        names = _run_twice(run, outs)
    _assert_kernels(names, 1, "v4")
    for (t, rows, K, Kh, hidden, logits), ref in zip(args, refs):
        hidden.check_guard("disc hidden")
        logits.check_guard("disc logits")
        _check_tiles(f"split + strided: disc hidden {rows}x{Kh}x{K}", hidden.t, ref)


# ------------------------------------------------------------------------------------------------
# operator entry points: the real epilogues and multi-group plans
# ------------------------------------------------------------------------------------------------
def _scale(p):
    import numpy as np
    return float(np.float32(1.0) / (np.float32(1.0) - np.float32(p)))


@pytest.mark.parametrize("scratch", [False, True], ids=["nosplit", "split"])
@pytest.mark.parametrize("F", [512, 1100, 255])
@pytest.mark.parametrize("D", [2048, 2044])
def test_x3_shared_layer_is_fp32_grade(D, F, scratch):
    """ta3n_shared_fc_fwd: relu(x W^T + b), without dropout, with RNG dropout (p = 0.3, the masks rebuilt by
    oracle/dropout_rng) and with a uint8 keep mask (the generic epilogue; split: the scalar reduce)."""
    from oracle import dropout_rng as drng
    from ta3n_b200 import _lib
    lib = _lib.load()
    dev, st, p = _dev(), torch.cuda.current_stream().cuda_stream, 0.3
    g = torch.Generator().manual_seed(D + F)
    W = torch.randn(F, D, generator=g) / D ** 0.5
    b = 0.1 * torch.randn(F, generator=g)
    dW, db = W.to(dev), b.to(dev)
    for rows_s, rows_t in [(450, 250), (333, 0)]:
        rows = rows_s + rows_t
        shapes = [(r, F, D) for r in (rows_s, rows_t) if r > 0]
        ks = _regime(shapes, scratch)[0]
        if scratch:
            assert max(ks) > 1, f"rows {rows_s}+{rows_t}: the planner no longer splits K ({ks})"
        xs = torch.randn(rows_s, D, generator=g)
        xt = torch.randn(rows_t, D, generator=g)
        x = torch.cat([xs, xt])
        pre = torch.relu(_mm(x, W) + b.double())
        dxs, dxt = xs.to(dev), (xt.to(dev) if rows_t else None)
        keep8 = (torch.rand(rows, F, generator=g) < 0.7).to(torch.uint8)
        dkeep = keep8.to(dev)
        m = drng.shared_masks(SEED, 0, rows_s, rows_t, 1, F, p)
        rng_keep = torch.cat([m["i_source"], m["i_target"]])
        for mode in ("none", "rng", "mask"):
            if mode == "none":
                drop, ref, vec = _lib.Dropout(0.0, None, 0, None), pre, True
            elif mode == "rng":
                drop, ref, vec = _lib.Dropout(p, None, SEED, None), pre * rng_keep.double() * _scale(p), True
            else:
                drop, ref, vec = _lib.Dropout(p, dkeep.data_ptr(), 0, None), pre * keep8.double() * _scale(p), False
            feat = _Out(rows, F)
            run = lambda: _lib.check(lib.ta3n_shared_fc_fwd(  # noqa: E731
                dxs.data_ptr(), rows_s, None if dxt is None else dxt.data_ptr(), rows_t, D, dW.data_ptr(),
                db.data_ptr(), F, C.byref(drop), feat.ptr(), st))
            with _Scratch(scratch):
                names = _run_twice(run, [feat])
            _assert_kernels(names, 1, _reduce_kind(ks, vec and F % 4 == 0))
            feat.check_guard("shared feat")
            _check_tiles(f"shared D={D} F={F} rows={rows_s}+{rows_t} drop={mode} ksplit={ks}", feat.t, ref)


@pytest.mark.parametrize("scratch", [False, True], ids=["nosplit", "split"])
@pytest.mark.parametrize("F", [512, 1100])
@pytest.mark.parametrize("T", [5, 9, 10])
def test_x3_forward_batch_disc_and_trn_is_fp32_grade(T, F, scratch):
    """ta3n_fwd_batch_begin -> ta3n_disc_fwd + ta3n_trn_fwd(relu_input=0) -> flush: the frame discriminator's hidden
    layer and every TRN relation in one precise plan.  T = 10 has 143 segments: the plan is cut into two launches.
    F = 1100 makes every segment end on a ragged slab."""
    from oracle import ta3n_oracle as orc
    from ta3n_b200 import _lib
    from ta3n_b200.functional import relation_set
    lib = _lib.load()
    dev, st = _dev(), torch.cuda.current_stream().cuda_stream
    M, H = 37, 256                      # videos; frame rows M * T
    rs = relation_set(T)
    tuples = orc.relation_tuples(T)
    R = T - 1
    assert (rs.n_slots + 1 > MAX_SEGS) == (T == 10), rs.n_slots     # the TRN's segments and the discriminator's
    g = torch.Generator().manual_seed(T * 100 + F)
    x = torch.randn(M * T, F, generator=g)
    W1 = torch.randn(F, F, generator=g) / F ** 0.5
    b1 = 0.1 * torch.randn(F, generator=g)
    W2 = torch.randn(2, F, generator=g) / F ** 0.5
    b2 = torch.randn(2, generator=g)
    Ws = [torch.randn(H, s * F, generator=g) / (s * F) ** 0.5 for s in range(T, 1, -1)]
    bs = [0.1 * torch.randn(H, generator=g) for _ in range(R)]
    ref_hidden = torch.relu(_mm(x, W1) + b1.double())
    xv = x.view(M, T, F)
    ref_act = []
    for i, rels in enumerate(tuples):
        for tup in rels:
            ref_act.append(torch.relu(_mm(xv[:, list(tup), :].reshape(M, -1), Ws[i]) + bs[i].double()))
    ref_act = torch.stack(ref_act)
    d = {k: v.to(dev) for k, v in dict(x=x, W1=W1, b1=b1, W2=W2, b2=b2).items()}
    dWs, dbs = [w.to(dev) for w in Ws], [v.to(dev) for v in bs]
    hidden, logits = _Out(M * T, F), _Out(M * T, 2)
    act, feat_rel = _Out(rs.n_rel, M, H), _Out(M, R, H)
    wp, bp = _lib.ptr_array([w.data_ptr() for w in dWs]), _lib.ptr_array([v.data_ptr() for v in dbs])

    def run():
        _lib.check(lib.ta3n_fwd_batch_begin())
        _lib.check(lib.ta3n_disc_fwd(d["x"].data_ptr(), M * T, F, F, d["W1"].data_ptr(), d["b1"].data_ptr(),
                                     d["W2"].data_ptr(), d["b2"].data_ptr(), hidden.ptr(), logits.ptr(), st))
        _lib.check(lib.ta3n_trn_fwd(d["x"].data_ptr(), M, F, H, rs.ref, wp, bp, 0, act.ptr(), feat_rel.ptr(), st))
        _lib.check(lib.ta3n_fwd_batch_flush(None, 0, st))

    with _Scratch(scratch):
        names = _run_twice(run, [hidden, logits, act, feat_rel])
    launches = 2 if T == 10 else 1
    splits = any("splitk_reduce" in n for n in names)
    _assert_kernels(names, launches, "v4" if splits else None)
    for o, w in ((hidden, "hidden"), (logits, "logits"), (act, "act"), (feat_rel, "feat_rel")):
        o.check_guard(w)
    tag = f"T={T} F={F} {'split' if splits else 'unsplit'}"
    _check_tiles(f"fwd batch {tag}: disc hidden", hidden.t, ref_hidden)
    _check_tiles(f"fwd batch {tag}: TRN act ({rs.n_rel} relations)", act.t, ref_act)


@pytest.mark.parametrize("R", [4, 8, 19])
def test_x3_relation_discriminators_are_fp32_grade(R):
    """ta3n_relattn_fwd: relation i's hidden layer reads feat_rel[:, i, :] (a strided A, lda = R * H); the row kernel
    behind it (logits, entropy attention, pooling) at the row-kernel bound."""
    from oracle import ta3n_oracle as orc
    from ta3n_b200 import _lib
    lib = _lib.load()
    dev, st = _dev(), torch.cuda.current_stream().cuda_stream
    M, H = 300, 256
    g = torch.Generator().manual_seed(R)
    feat_rel = torch.randn(M, R, H, generator=g)
    W1 = [torch.randn(H, H, generator=g) / H ** 0.5 for _ in range(R)]
    b1 = [0.1 * torch.randn(H, generator=g) for _ in range(R)]
    W2 = [torch.randn(2, H, generator=g) / H ** 0.5 for _ in range(R)]
    b2 = [torch.randn(2, generator=g) for _ in range(R)]
    hid = torch.stack([torch.relu(_mm(feat_rel[:, i], W1[i]) + b1[i].double()) for i in range(R)])
    pred = torch.stack([hid[i] @ W2[i].double().t() + b2[i].double() for i in range(R)], 1)
    w = orc.entropy_attention(pred.reshape(-1, 2)).view(M, R)
    fv = ((w.unsqueeze(-1) + 1) * feat_rel.double()).sum(1)
    dfr = feat_rel.to(dev)
    dev_lists = [[t.to(dev) for t in lst] for lst in (W1, b1, W2, b2)]
    ptrs = [_lib.ptr_array([t.data_ptr() for t in lst]) for lst in dev_lists]
    hidden, pred_rel, attn, feat_video = _Out(R, M, H), _Out(M, R, 2), _Out(M, R), _Out(M, H)
    run = lambda: _lib.check(lib.ta3n_relattn_fwd(  # noqa: E731
        dfr.data_ptr(), M, R, H, *ptrs, 1, hidden.ptr(), pred_rel.ptr(), attn.ptr(), feat_video.ptr(), st))
    names = _run_twice(run, [hidden, pred_rel, attn, feat_video])
    _assert_kernels(names, 1, None)
    for o, what in ((hidden, "hidden"), (pred_rel, "pred_rel"), (attn, "attn"), (feat_video, "feat_video")):
        o.check_guard(what)
    _check_tiles(f"relattn R={R}: hidden", hidden.t, hid)
    for got, ref, what in ((pred_rel.t, pred, "pred_rel"), (attn.t, w, "attn"), (feat_video.t, fv, "feat_video")):
        err = _rel(got, ref)
        assert err < ROW_TOL, f"relattn R={R} {what}: normwise rel err {err:.2e}"


def test_x3_general_attention_is_fp32_grade():
    """ta3n_general_attn_fwd: the hidden layer has a bias and no ReLU (EPI_BIAS alone: the precise kernel's generic
    epilogue); tanh, the softmax over the relations and the weighted sum added onto feat_video follow in a row
    kernel."""
    from ta3n_b200 import _lib
    lib = _lib.load()
    dev, st = _dev(), torch.cuda.current_stream().cuda_stream
    M, R, H = 300, 8, 256
    g = torch.Generator().manual_seed(1)
    feat_rel = torch.randn(M * R, H, generator=g)
    W1 = torch.randn(H, H, generator=g) / H ** 0.5
    b1 = 0.1 * torch.randn(H, generator=g)
    w2 = torch.randn(1, H, generator=g) / H ** 0.5
    b2 = torch.randn(1, generator=g)
    fv0 = torch.randn(M, H, generator=g)
    pre = _mm(feat_rel, W1) + b1.double()
    hid = torch.tanh(pre)
    a = torch.softmax((hid @ w2.double().t() + b2.double()).view(M, R), 1)
    fv = fv0.double() + (a.unsqueeze(-1) * feat_rel.double().view(M, R, H)).sum(1)
    d = [t.to(dev) for t in (feat_rel, W1, b1, w2, b2)]
    hidden, attn, feat_video = _Out(M * R, H), _Out(M, R), _Out(M, H)
    dfv0 = fv0.to(dev)

    def run():
        feat_video.t.copy_(dfv0)
        _lib.check(lib.ta3n_general_attn_fwd(d[0].data_ptr(), M, R, H, *[t.data_ptr() for t in d[1:]],
                                             hidden.ptr(), attn.ptr(), feat_video.ptr(), st))

    names = _run_twice(run, [hidden, attn, feat_video])
    _assert_kernels(names, 1, None)
    for o, what in ((hidden, "hidden"), (attn, "attn"), (feat_video, "feat_video")):
        o.check_guard(what)
    _check_tiles("general attention: tanh(hidden)", hidden.t, hid)
    for got, ref, what in ((attn.t, a, "attn"), (feat_video.t, fv, "feat_video")):
        err = _rel(got, ref)
        assert err < ROW_TOL, f"general attention {what}: normwise rel err {err:.2e}"


# ------------------------------------------------------------------------------------------------
# the other operand layouts
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,N,K", [(200, 136, 2000), (256, 256, 1024), (64, 64, 4104)])
def test_x3_mn_major_operands_are_fp32_grade(M, N, K):
    import ta3n_b200
    from ta3n_b200 import _lib
    lib = _lib.load()
    ta3n_b200.set_gemm_engine("tf32x3")
    g = torch.Generator().manual_seed(M + 5 * N + 11 * K)
    A = torch.randn(M, K, generator=g)
    B = torch.randn(K, N, generator=g)
    ref = A.double() @ B.double()
    dev = torch.device("cuda:0")
    At = A.t().contiguous().to(dev)          # M-major: A(m, k) = At[k * M + m]
    Bn = B.contiguous().to(dev)              # N-major: B(k, n) = Bn[k * N + n]
    C = torch.full((M, N), 7.0, device=dev)
    _lib.timing_enable(True)
    try:
        _lib.check(lib.ta3n_gemm_ex(At.data_ptr(), M, 0, Bn.data_ptr(), N, 0, C.data_ptr(), N, M, N, K, None, 0,
                                    torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        sites = _lib.timing_report()
    finally:
        _lib.timing_enable(False)
    assert "wgrad_small_x3" in sites, f"the precise kernel did not run: {sorted(sites)}"
    err = _rel(C, ref)
    assert err < X3_TOL, f"M-major x N-major precise GEMM {M}x{N}x{K}: normwise rel err {err:.2e}"


_DGRAD_CHILD = r"""
import json, sys
import torch
import ta3n_b200
from ta3n_b200 import _lib
lib = _lib.load()
ta3n_b200.set_gemm_engine("tf32x3")
rows, K, Kh, beta = 300, 2048, 900, 0.5          # GEMM: M = 300, N = 2048, K = 900 (29 slabs, ragged)
g = torch.Generator().manual_seed(7)
x = torch.randn(rows, K, generator=g)
W1 = torch.randn(Kh, K, generator=g) / K ** 0.5
W2 = torch.randn(2, Kh, generator=g)
hidden = torch.randn(rows, Kh, generator=g)
g_logits = torch.randn(rows, 2, generator=g)
dev = torch.device("cuda:0")
t = {k: v.to(dev) for k, v in dict(x=x, W1=W1, W2=W2, hidden=hidden, g=g_logits).items()}
dx = torch.empty(rows, K, device=dev)
dW1, db1 = torch.empty(Kh, K, device=dev), torch.empty(Kh, device=dev)
dW2, db2 = torch.empty(2, Kh, device=dev), torch.empty(2, device=dev)
nbytes = lib.ta3n_disc_bwd_workspace_bytes(rows, K, Kh)
ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
_lib.check(lib.ta3n_disc_bwd(t["x"].data_ptr(), rows, K, Kh, t["W1"].data_ptr(), t["W2"].data_ptr(),
                             t["hidden"].data_ptr(), t["g"].data_ptr(), beta, dx.data_ptr(), 0, dW1.data_ptr(),
                             db1.data_ptr(), dW2.data_ptr(), db2.data_ptr(), ws.data_ptr(), nbytes,
                             torch.cuda.current_stream().cuda_stream))
torch.cuda.synchronize()
dH = (g_logits.double() @ W2.double()) * (hidden > 0).double()
ref = -beta * dH @ W1.double()
err = ((dx.double().cpu() - ref).norm() / ref.norm()).item()
print(json.dumps({"err": err}))
"""


def test_x3_dgrad_k_major_x_n_major_is_fp32_grade():
    env = dict(os.environ, TA3N_X3_DGRAD="1", PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _DGRAD_CHILD]
    res = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout + res.stderr
    err = json.loads(res.stdout.strip().splitlines()[-1])["err"]
    assert err < X3_TOL, f"K-major x N-major precise data gradient: normwise rel err {err:.2e}"
