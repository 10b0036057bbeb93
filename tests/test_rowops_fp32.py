"""The row kernels (csrc/rowops.cuh), the step program's row kernels (csrc/step_rows.cuh) and the loss kernels at fp32
grade, against fp64 restatements of the same operators.

These kernels do fp32 arithmetic only, so with the ReLU pattern pinned they must agree with fp64 to rounding.  One rule
holds for the whole file: for every tensor,

    ||cuda - ref64|| <= TOL_FP32 * ||ref64|| + 8 * noise,   noise = max(||ref32 - ref64||, 4 ulp * ||summands||)

where ref32 is the same restatement run in fp32 on the CPU.  The rule is applied per tensor and per slice: per row of an
[M, *] output, per relation of [M, R, *] and [R, M, H] tensors, per class row of a classifier's weight gradient, so
that one wrong row or relation cannot hide in the norm of the rest.

Operators run one at a time through the C ABI under the exact fp32 GEMM engine (a tf32 GEMM error must not hide a
row-kernel error), with outputs NaN-filled behind guard regions that must stay untouched.  The loss terms are checked
each alone and at full weight (gamma = 1 as well as the shipped 0.003), so the attentive entropy's gradient is not
hidden at 0.3 % of a tensor.  The training step is checked whole at gamma = 1 and 0.003 on the activation pattern it
realised: the only way to reach the step program's row kernels, which have no entry points of their own.
"""
import ctypes as C
import math
import random

import pytest
import torch
import torch.nn.functional as F

from oracle import mcd_oracle as mcd
from oracle import ta3n_oracle as orc
from tests.golden_util import TOL_FP32

pytestmark = pytest.mark.gpu

EPS32 = 2.0 ** -24
ULPS = 4.0
_WORST = []


def _dev():
    return torch.device("cuda:0")


@pytest.fixture(autouse=True)
def fp32_engine(request):
    """Every test runs under the exact fp32 GEMM engine unless it selects another; the worst error / bound ratio
    of the test is printed at its end."""
    import ta3n_b200
    ta3n_b200.set_gemm_engine("fp32")
    _WORST.clear()
    yield
    ta3n_b200.set_gemm_engine("tf32x3")
    if _WORST:
        print(f"\n[fp32-grade] {request.node.name}: worst error/bound {max(_WORST):.3f}")


def _h(t):
    return t.detach().double().cpu()


def _slice_norms(t, dim):
    return t.movedim(dim, 0).reshape(t.shape[dim], -1).norm(dim=1)


def check(what, got, r64, r32, dims=(), scale=None, tol=TOL_FP32, noise_scale=1.0):
    """got vs the fp64 reference under the file's rule, for the whole tensor and for each slice along ``dims``.
    ``scale``: magnitude of the summands behind each element (default |ref64|), for the ulp floor of sums that
    cancel."""
    got, r64, r32 = _h(got), _h(r64), _h(r32)
    assert got.shape == r64.shape == r32.shape, (what, got.shape, r64.shape, r32.shape)
    assert bool(torch.isfinite(got).all()), f"{what}: non-finite entries (an output element left unwritten?)"
    s = r64.abs() if scale is None else _h(scale).abs().expand_as(r64)
    diff, err32 = got - r64, r32 - r64

    def rule(d, den, n32, sc, label):
        noise = torch.maximum(n32, ULPS * EPS32 * sc) * noise_scale
        bound = tol * den + 8.0 * noise
        bad = d > bound
        if bool(bad.any()):
            i = int(torch.nonzero(bad)[0, 0]) if d.dim() else 0
            dd, bb = (d[i], bound[i]) if d.dim() else (d, bound)
            raise AssertionError(f"{what}{label}{'' if not d.dim() else f' slice {i}'}: ||diff|| {float(dd):.3e} > "
                                 f"bound {float(bb):.3e} (tol {tol:.0e})")
        ratio = torch.where(bound > 0, d / bound.clamp_min(1e-300), torch.zeros_like(d))
        return float(ratio.max()) if ratio.dim() else float(ratio)

    worst = rule(diff.norm(), r64.norm(), err32.norm(), s.norm(), "")
    for dim in dims:
        worst = max(worst, rule(_slice_norms(diff, dim), _slice_norms(r64, dim), _slice_norms(err32, dim),
                                _slice_norms(s, dim), f" [dim {dim}]"))
    _WORST.append(worst)
    return worst


class Buf:
    """A device buffer of ``shape`` at float offset ``off`` inside a larger allocation whose guard regions (and, unless
    ``init`` is given, the buffer itself) hold NaN.  ``off`` = 1 makes the buffer 4-byte but not 16-byte aligned."""

    def __init__(self, *shape, init=None, off=64):
        n = math.prod(shape)
        self.full = torch.full((n + off + 64,), float("nan"), device=_dev())
        self.off, self.n = off, n
        self.t = self.full[off:off + n].view(*shape)
        if init is not None:
            self.t.copy_(init.reshape(shape))

    @property
    def p(self):
        return self.t.data_ptr()

    def cpu(self):
        return self.t.detach().cpu()

    def guards_intact(self):
        g = torch.cat([self.full[:self.off], self.full[self.off + self.n:]])
        return bool(torch.isnan(g).all())


def _guards(*bufs):
    for b in bufs:
        if b is not None:
            assert b.guards_intact(), "a write landed outside its output"


def _ws(nbytes):
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=_dev())


def _st():
    return torch.cuda.current_stream().cuda_stream


def _lib():
    from ta3n_b200 import _lib as L
    return L, L.load()


def _pa(ptrs):
    from ta3n_b200._lib import ptr_array
    return ptr_array(ptrs)


def _ref(fn, *args):
    """Run the restatement ``fn(dtype, *args)`` in fp64 and in fp32 on the CPU."""
    return fn(torch.float64, *args), fn(torch.float32, *args)


def _leaf(t, dt):
    return t.detach().to(dt).clone().requires_grad_(True)


def _grads(out, inputs, allow_unused=False):
    return torch.autograd.grad(out, inputs, allow_unused=allow_unused)


# ================================================================================================
# 1. operators one by one through the C ABI
# ================================================================================================
def _relattn_inputs(M, R, H, seed):
    g = torch.Generator().manual_seed(seed)
    fr = torch.rand(M, R, H, generator=g) * 2.0
    W1 = [torch.randn(H, H, generator=g) / math.sqrt(H) for _ in range(R)]
    b1 = [0.1 * torch.randn(H, generator=g) for _ in range(R)]
    W2 = [2.0 * torch.randn(2, H, generator=g) / math.sqrt(H) for _ in range(R)]
    b2 = [0.3 * torch.randn(2, generator=g) for _ in range(R)]
    G = torch.randn(M, H, generator=g)
    gp = torch.randn(M, R, 2, generator=g)
    ga = torch.randn(M, R, generator=g)
    attn_ext = torch.rand(M, R, generator=g)
    return fr, W1, b1, W2, b2, G, gp, ga, attn_ext


def _relattn_ref(dt, fr, W1, b1, W2, b2, gates, use_attn, beta, attn_ext, G, gp, ga):
    """relation discriminators (GRL -> Linear -> ReLU -> Linear) + attention + pooling, and the gradient of
    <G, feat_video> + <gp, pred_rel> + <ga, attn>; the ReLU pattern is ``gates`` (see orc._relu)."""
    R = fr.shape[1]
    x = _leaf(fr, dt)
    w1, bb1, w2, bb2 = ([_leaf(t, dt) for t in L] for L in (W1, b1, W2, b2))
    z = [F.linear(orc.grad_reverse(x[:, i], beta), w1[i], bb1[i]) for i in range(R)]
    hid = [orc._relu(z[i], gates[i]) for i in range(R)]
    pred = torch.stack([F.linear(hid[i], w2[i], bb2[i]) for i in range(R)], 1)
    if use_attn == 1:
        attn = orc.entropy_attention(pred.reshape(-1, 2)).view(-1, R)
        fv = ((attn + 1).unsqueeze(-1) * x).sum(1)
    elif use_attn == 0:
        attn = x[:, :, 0]
        fv = x.sum(1)
    else:
        attn = attn_ext.to(dt)
        fv = ((attn + 1).unsqueeze(-1) * x).sum(1)
    loss = (fv * G.to(dt)).sum()
    if gp is not None:
        loss = loss + (pred * gp.to(dt)).sum()
    if ga is not None and use_attn != 2:
        loss = loss + (attn * ga.to(dt)).sum()
    ins = [x, *w1, *bb1, *w2, *bb2, pred, *z]
    gr = _grads(loss, ins, allow_unused=True)            # without g_pred_rel the second layers get no gradient
    d = iter(torch.zeros_like(t) if g is None else g for g, t in zip(gr, ins))
    out = dict(hidden=torch.stack(hid).detach(), pred_rel=pred.detach(), attn=attn.detach(), feat_video=fv.detach(),
               d_feat_rel=next(d))
    out["dW1"] = torch.stack([next(d) for _ in range(R)])
    out["db1"] = torch.stack([next(d) for _ in range(R)])
    out["dW2"] = torch.stack([next(d) for _ in range(R)])
    out["db2"] = torch.stack([next(d) for _ in range(R)])
    dpred = next(d)
    dz = torch.stack([next(d) for _ in range(R)])
    out["scale_db2"] = dpred.abs().sum(0)                # [R, 2]: summands of the bias gradients
    out["scale_db1"] = dz.abs().sum(1)                   # [R, H]
    return out


def _run_relattn(M, R, H, use_attn, with_gp, with_ga, seed):
    L, lib = _lib()
    fr, W1, b1, W2, b2, G, gp, ga, attn_ext = _relattn_inputs(M, R, H, seed)
    dev = lambda ts: [t.to(_dev()) for t in ts]          # noqa: E731
    W1d, b1d, W2d, b2d = dev(W1), dev(b1), dev(W2), dev(b2)
    frb = Buf(M, R, H, init=fr.to(_dev()))
    hid, pred, attn, fv = Buf(R, M, H), Buf(M, R, 2), Buf(M, R), Buf(M, H)
    ptrs = lambda ts: _pa([t.data_ptr() for t in ts])    # noqa: E731
    L.check(lib.ta3n_relattn_fwd(frb.p, M, R, H, ptrs(W1d), ptrs(b1d), ptrs(W2d), ptrs(b2d), 1 if use_attn == 1 else 0,
                                 hid.p, pred.p, attn.p, fv.p, _st()))
    if use_attn == 2:                                    # weights made elsewhere ('general'): the caller's buffer
        attn.t.copy_(attn_ext.to(_dev()))
    beta = 0.6
    Gb = Buf(M, H, init=G.to(_dev()))
    gpb = Buf(M, R, 2, init=gp.to(_dev())) if with_gp else None
    gab = Buf(M, R, init=ga.to(_dev())) if with_ga else None
    dfr = Buf(M, R, H)
    dW1, db1, dW2, db2 = Buf(R, H, H), Buf(R, H), Buf(R, 2, H), Buf(R, 2)
    ws = _ws(lib.ta3n_relattn_bwd_workspace_bytes(M, R, H))
    rows = lambda b, n: _pa([b.p + 4 * i * n for i in range(R)])   # noqa: E731
    L.check(lib.ta3n_relattn_bwd(frb.p, M, R, H, ptrs(W1d), ptrs(W2d), use_attn, hid.p, pred.p, attn.p, Gb.p,
                                 None if gpb is None else gpb.p, None if gab is None else gab.p, beta, dfr.p,
                                 rows(dW1, H * H), rows(db1, H), rows(dW2, 2 * H), rows(db2, 2), ws.data_ptr(),
                                 ws.numel(), _st()))
    torch.cuda.synchronize()
    gates = [(h > 0) for h in hid.cpu()]
    args = (fr, W1, b1, W2, b2, gates, use_attn, beta, attn_ext, G, gp if with_gp else None, ga if with_ga else None)
    r64, r32 = _ref(_relattn_ref, *args)
    check("hidden", hid.t, r64["hidden"], r32["hidden"], dims=(0, 1))
    check("pred_rel", pred.t, r64["pred_rel"], r32["pred_rel"], dims=(0, 1))
    if use_attn != 2:
        check("attn", attn.t, r64["attn"], r32["attn"], dims=(0, 1))
        check("feat_video", fv.t, r64["feat_video"], r32["feat_video"], dims=(0,))
    check("d_feat_rel", dfr.t, r64["d_feat_rel"], r32["d_feat_rel"], dims=(0, 1))
    check("dW1", dW1.t, r64["dW1"], r32["dW1"], dims=(0,))
    check("db1", db1.t, r64["db1"], r32["db1"], dims=(0,), scale=r64["scale_db1"])
    check("dW2", dW2.t, r64["dW2"], r32["dW2"], dims=(0,))
    check("db2", db2.t, r64["db2"], r32["db2"], dims=(0,), scale=r64["scale_db2"])
    _guards(hid, pred, attn, fv, dfr, dW1, db1, dW2, db2)


@pytest.mark.parametrize("use_attn", [0, 1, 2])
@pytest.mark.parametrize("R,H", [(1, 256), (8, 256), (9, 256), (17, 256), (32, 256), (1, 250), (8, 250), (9, 250),
                                 (17, 250), (32, 250), (1, 1100), (9, 1100), (17, 1100)])
def test_relattn_fwd_bwd(R, H, use_attn):
    """ta3n_relattn_fwd / _bwd: R relations over kRelWarps = 8 warps (one pass, several, a partial last one; R = 32
    is the documented limit and gives more than 40 column-sum jobs), widths on and off the float4 grid and above
    1024, and use_attn 'none' / TransAttn / weights from 'general' attention."""
    _run_relattn(7, R, H, use_attn, True, True, seed=R * 31 + H + use_attn)


@pytest.mark.parametrize("use_attn", [0, 1, 2])
@pytest.mark.parametrize("with_gp,with_ga", [(False, False), (True, False), (False, True)])
def test_relattn_bwd_optional_gradients(with_gp, with_ga, use_attn):
    """g_pred_rel and g_attn NULL and non-NULL."""
    _run_relattn(13, 9, 256, use_attn, with_gp, with_ga, seed=7 + 2 * with_gp + with_ga)


def _general_ref(dt, fr, W1, b1, w2, b2, S0, D0, G, ga):
    """softmax_r(w2 tanh(W1 feat_rel + b1) + b2) and the plain sum S0 + sum_r a_r feat_rel_r; the gradient through the
    weights only (the (a + 1) G part is ta3n_relattn_bwd's), added to D0."""
    M, R, H = fr.shape
    x = _leaf(fr, dt)
    p = {"attn_layer.0.weight": _leaf(W1, dt), "attn_layer.0.bias": _leaf(b1, dt), "attn_layer.2.weight": _leaf(w2, dt),
         "attn_layer.2.bias": _leaf(b2, dt)}
    hid = torch.tanh(F.linear(x.reshape(-1, H), p["attn_layer.0.weight"], p["attn_layer.0.bias"]))
    a = orc.general_attention(p, x)
    fv = S0.to(dt) + (a.detach().unsqueeze(-1) * x.detach()).sum(1)
    loss = (G.to(dt) * (a.unsqueeze(-1) * x.detach()).sum(1)).sum()
    if ga is not None:
        loss = loss + (ga.to(dt) * a).sum()
    gx, gW1, gb1, gw2, gb2 = _grads(loss, [x, *p.values()])
    return dict(hidden=hid.detach(), attn=a.detach(), feat_video=fv, d_feat_rel=D0.to(dt) + gx, dW1=gW1, db1=gb1,
                dw2=gw2, db2=gb2)


@pytest.mark.parametrize("with_ga", [True, False])
@pytest.mark.parametrize("R", [1, 9, 32])
def test_general_attn_fwd_bwd(R, with_ga):
    L, lib = _lib()
    M, H = 11, 256
    g = torch.Generator().manual_seed(40 + R)
    fr = torch.rand(M, R, H, generator=g) * 2
    W1, b1 = torch.randn(H, H, generator=g) / math.sqrt(H), 0.1 * torch.randn(H, generator=g)
    w2, b2 = 3 * torch.randn(1, H, generator=g) / math.sqrt(H), torch.randn(1, generator=g)
    S0, D0, G = torch.randn(M, H, generator=g), torch.randn(M, R, H, generator=g), torch.randn(M, H, generator=g)
    ga = torch.randn(M, R, generator=g) if with_ga else None
    d = lambda t: t.to(_dev())                            # noqa: E731
    frb = Buf(M, R, H, init=d(fr))
    W1d, b1d, w2d, b2d = d(W1), d(b1), d(w2), d(b2)
    hid, attn, fv = Buf(M * R, H), Buf(M, R), Buf(M, H, init=d(S0))
    L.check(lib.ta3n_general_attn_fwd(frb.p, M, R, H, W1d.data_ptr(), b1d.data_ptr(), w2d.data_ptr(), b2d.data_ptr(),
                                      hid.p, attn.p, fv.p, _st()))
    dfr = Buf(M, R, H, init=d(D0))
    dW1, db1, dw2, db2 = Buf(H, H), Buf(H), Buf(1, H), Buf(1)
    gab = None if ga is None else Buf(M, R, init=d(ga))
    Gb = Buf(M, H, init=d(G))
    ws = _ws(lib.ta3n_general_attn_bwd_workspace_bytes(M, R, H))
    L.check(lib.ta3n_general_attn_bwd(frb.p, M, R, H, W1d.data_ptr(), w2d.data_ptr(), hid.p, attn.p, Gb.p,
                                      None if gab is None else gab.p, dfr.p, dW1.p, db1.p, dw2.p, db2.p,
                                      ws.data_ptr(), ws.numel(), _st()))
    torch.cuda.synchronize()
    r64, r32 = _ref(_general_ref, fr, W1, b1, w2, b2, S0, D0, G, ga)
    check("hidden", hid.t.view(M, R, H), r64["hidden"].view(M, R, H), r32["hidden"].view(M, R, H), dims=(0, 1))
    check("attn", attn.t, r64["attn"], r32["attn"], dims=(0, 1))
    check("feat_video", fv.t, r64["feat_video"], r32["feat_video"], dims=(0,))
    check("d_feat_rel", dfr.t, r64["d_feat_rel"], r32["d_feat_rel"], dims=(0, 1))
    if R > 1:
        check("dW1", dW1.t, r64["dW1"], r32["dW1"], dims=(0,))
        check("db1", db1.t, r64["db1"], r32["db1"])
        check("dw2", dw2.t, r64["dw2"], r32["dw2"])
    else:                                                # one relation: the softmax is constant, nothing flows
        for b in (dW1, db1, dw2):
            assert bool((b.cpu() == 0).all())
    # db2 shifts every logit of the softmax alike: zero up to rounding
    assert abs(float(db2.cpu()[0])) <= 1e-5 * max(1.0, float(r64["dw2"].norm()))
    _guards(hid, attn, fv, dfr, dW1, db1, dw2, db2)


def _frame_attn_ref(dt, feat, logits, D, G0):
    x, lg = _leaf(feat, dt), _leaf(logits, dt)
    w = orc.entropy_attention(lg)
    out = (w.unsqueeze(-1) + 1) * x
    gx, gl = _grads((out * D.to(dt)).sum(), [x, lg])
    return dict(out=out.detach(), d_feat=gx, g_logits=G0.to(dt) + gl)


@pytest.mark.parametrize("rows,Fd", [(1000, 512), (333, 250)])
def test_frame_attn_fwd_bwd(rows, Fd):
    """ta3n_frame_attn_fwd / _bwd, with a third of the rows' logits saturated (|delta| of 30 to 80)."""
    L, lib = _lib()
    g = torch.Generator().manual_seed(rows)
    feat = torch.rand(rows, Fd, generator=g)
    logits = torch.randn(rows, 2, generator=g)
    logits[::3] *= 40.0
    logits[::3, 0] += torch.sign(logits[::3, 0]) * 30.0
    D, G0 = torch.randn(rows, Fd, generator=g), torch.randn(rows, 2, generator=g)
    fb, lb = Buf(rows, Fd, init=feat.to(_dev())), Buf(rows, 2, init=logits.to(_dev()))
    out = Buf(rows, Fd)
    L.check(lib.ta3n_frame_attn_fwd(fb.p, lb.p, rows, Fd, out.p, _st()))
    dout, gl = Buf(rows, Fd, init=D.to(_dev())), Buf(rows, 2, init=G0.to(_dev()))
    L.check(lib.ta3n_frame_attn_bwd(fb.p, lb.p, rows, Fd, dout.p, gl.p, _st()))
    torch.cuda.synchronize()
    r64, r32 = _ref(_frame_attn_ref, feat, logits, D, G0)
    check("out", out.t, r64["out"], r32["out"], dims=(0,))
    check("d_feat", dout.t, r64["d_feat"], r32["d_feat"], dims=(0,))
    check("g_logits", gl.t, r64["g_logits"], r32["g_logits"], dims=(0,))
    _guards(out, dout, gl)


@pytest.mark.parametrize("M,T,Fd", [(37, 5, 250), (9, 33, 512)])
def test_segment_mean_fwd_bwd(M, T, Fd):
    L, lib = _lib()
    g = torch.Generator().manual_seed(T)
    x, gv = torch.randn(M, T, Fd, generator=g), torch.randn(M, Fd, generator=g)
    xb, gb = Buf(M, T, Fd, init=x.to(_dev())), Buf(M, Fd, init=gv.to(_dev()))
    out, dx = Buf(M, Fd), Buf(M, T, Fd)
    L.check(lib.ta3n_segment_mean_fwd(xb.p, M, T, Fd, out.p, _st()))
    L.check(lib.ta3n_segment_mean_bwd(gb.p, M, T, Fd, dx.p, _st()))
    torch.cuda.synchronize()
    ref = lambda dt: (x.to(dt).sum(1) / T, (gv.to(dt) / T).unsqueeze(1).expand(M, T, Fd))   # noqa: E731
    (o64, d64), (o32, d32) = ref(torch.float64), ref(torch.float32)
    check("mean", out.t, o64, o32, dims=(0,), scale=x.abs().sum(1) / T)
    check("dx", dx.t, d64, d32, dims=(0, 1))
    _guards(out, dx)


def test_grl_bwd_and_accumulate():
    """ta3n_grl_bwd (out = -beta g) and ta3n_accumulate with n not a multiple of 4 (float4 body + scalar tail)."""
    L, lib = _lib()
    g = torch.Generator().manual_seed(3)
    for n in (1001, 4099, 6):
        a, b = torch.randn(n, generator=g), torch.randn(n, generator=g)
        gb, out = Buf(n, init=a.to(_dev())), Buf(n)
        L.check(lib.ta3n_grl_bwd(gb.p, 0.75, out.p, n, _st()))
        dst = Buf(n, init=a.to(_dev()), off=64)
        src = Buf(n, init=b.to(_dev()), off=128)
        L.check(lib.ta3n_accumulate(dst.p, src.p, n, _st()))
        torch.cuda.synchronize()
        check(f"grl n={n}", out.t, -0.75 * a.double(), -0.75 * a)
        check(f"accumulate n={n}", dst.t, a.double() + b.double(), a + b, scale=a.abs() + b.abs())
        _guards(out, dst, src)


def _disc_ref(dt, x, W1, b1, W2, b2, gate, gl, beta, dx0):
    xx, w1, bb1, w2, bb2 = (_leaf(t, dt) for t in (x, W1, b1, W2, b2))
    z = F.linear(orc.grad_reverse(xx, beta), w1, bb1)
    h = orc._relu(z, gate)
    lo = F.linear(h, w2, bb2)
    gx, gw1, gb1, gw2, gb2, gz = _grads((lo * gl.to(dt)).sum(), [xx, w1, bb1, w2, bb2, z])
    return dict(hidden=h.detach(), logits=lo.detach(), dx=gx + (0 if dx0 is None else dx0.to(dt)), dW1=gw1, db1=gb1,
                dW2=gw2, db2=gb2, scale_db1=gz.abs().sum(0), scale_db2=gl.abs().sum(0).to(dt))


@pytest.mark.parametrize("accumulate", [0, 1])
@pytest.mark.parametrize("rows,K,off", [(300, 2048, 0), (600, 1024, 0), (600, 1024, 1), (4500, 250, 0),
                                        (4500, 256, 1)])
def test_disc_fwd_bwd(rows, K, off, accumulate):
    """ta3n_disc_fwd / _bwd (GRL + two-layer discriminator, Kh = K): rows above kHeadMaxK (2048), W2 in shared memory,
    more than 4224 rows (the grid-stride loop of head_fwd), and buffers one float off 16-byte alignment, which
    takes the scalar twins of head_bwd_data and of the column sums."""
    L, lib = _lib()
    g = torch.Generator().manual_seed(rows + K + off)
    x = torch.rand(rows, K, generator=g)
    W1, b1 = torch.randn(K, K, generator=g) / math.sqrt(K), 0.1 * torch.randn(K, generator=g)
    W2, b2 = torch.randn(2, K, generator=g) / math.sqrt(K), 0.1 * torch.randn(2, generator=g)
    gl = torch.randn(rows, 2, generator=g) / rows
    dx0 = torch.randn(rows, K, generator=g) if accumulate else None
    d = lambda t: Buf(*t.shape, init=t.to(_dev()), off=64 + off)   # noqa: E731
    xb, W1b, b1b, W2b, b2b, glb = d(x), d(W1), d(b1), d(W2), d(b2), d(gl)
    hid, lo = Buf(rows, K, off=64 + off), Buf(rows, 2, off=64 + off)
    L.check(lib.ta3n_disc_fwd(xb.p, rows, K, K, W1b.p, b1b.p, W2b.p, b2b.p, hid.p, lo.p, _st()))
    dx = d(dx0) if accumulate else Buf(rows, K, off=64 + off)
    dW1, db1, dW2, db2 = (Buf(*s, off=64 + off) for s in ((K, K), (K,), (2, K), (2,)))
    ws = _ws(lib.ta3n_disc_bwd_workspace_bytes(rows, K, K))
    beta = 0.7
    L.check(lib.ta3n_disc_bwd(xb.p, rows, K, K, W1b.p, W2b.p, hid.p, glb.p, beta, dx.p, accumulate, dW1.p, db1.p,
                              dW2.p, db2.p, ws.data_ptr(), ws.numel(), _st()))
    torch.cuda.synchronize()
    gate = hid.cpu() > 0
    r64, r32 = _ref(_disc_ref, x, W1, b1, W2, b2, gate, gl, beta, dx0)
    check("hidden", hid.t, r64["hidden"], r32["hidden"], dims=(0,))
    check("logits", lo.t, r64["logits"], r32["logits"], dims=(0,))
    check("dx", dx.t, r64["dx"], r32["dx"], dims=(0,))
    check("dW1", dW1.t, r64["dW1"], r32["dW1"], dims=(0,))
    check("db1", db1.t, r64["db1"], r32["db1"], scale=r64["scale_db1"])
    check("dW2", dW2.t, r64["dW2"], r32["dW2"], dims=(0,))
    check("db2", db2.t, r64["db2"], r32["db2"], scale=r64["scale_db2"])
    _guards(hid, lo, dx, dW1, db1, dW2, db2)


def _head_ref(dt, x, Wc, bc, keep, p, gpred, extra, gext, scale):
    xx, w, b = _leaf(x, dt), _leaf(Wc, dt), _leaf(bc, dt)
    dr = xx if keep is None else xx * keep.to(dt) / (1.0 - p)
    dr_h = dr.detach().requires_grad_(True)
    pred = F.linear(dr_h, w, b)
    gd, gw, gb = _grads((pred * gpred.to(dt)).sum(), [dr_h, w, b])
    # d_feat_video = ((g_pred Wc) + extra) * grad_scale, back through the dropout, + the external gradient
    gd = (gd + (0 if extra is None else extra.to(dt))) * scale
    gx = gd if keep is None else gd * keep.to(dt) / (1.0 - p)
    if gext is not None:
        gx = gx + gext.to(dt)
    return dict(dropped=dr.detach(), pred=pred.detach(), d_feat_video=gx, dWc=gw, dbc=gb,
                scale_dbc=gpred.abs().sum(0).to(dt))


HEAD_CASES = {
    # id: (M, H, C, dropout, extra and g_ext, d_feat_video NULL, grad_scale)
    "c2_h256": (150, 256, 2, False, False, False, 1.0),
    "c5_h256_drop_extra": (150, 256, 5, True, True, False, 1.0),
    "c33_h256_drop": (150, 256, 33, True, False, False, -0.7),
    "c200_h256_wsmem_out": (150, 256, 200, False, True, False, 1.0),
    "c12_h1100_drop_extra": (97, 1100, 12, True, True, False, -0.7),
    "c33_h1100": (97, 1100, 33, False, False, False, 1.0),
    "c12_h256_no_dfeat": (150, 256, 12, True, False, True, -0.7),
    "c200_h250": (61, 250, 200, True, True, False, -0.7),
}


@pytest.mark.parametrize("case", list(HEAD_CASES))
def test_video_head_fwd_bwd(case):
    """ta3n_video_head_fwd / _bwd: C = 2 / 5 (column-sum weight gradient in passes of 4), 33 and 200 (GEMM weight
    gradient; at H = 256, W of C = 200 no longer fits shared memory), H = 1100 above kHeadMaxK, mask dropout,
    d_dropped_extra / g_feat_video_ext present and absent, d_feat_video = NULL and grad_scale = -0.7."""
    L, lib = _lib()
    M, H, Cn, drop, ext, no_dfeat, scale = HEAD_CASES[case]
    g = torch.Generator().manual_seed(M + H + Cn)
    x = torch.rand(M, H, generator=g) * 2
    Wc, bc = torch.randn(Cn, H, generator=g) / math.sqrt(H), 0.1 * torch.randn(Cn, generator=g)
    keep = (torch.rand(M, H, generator=g) < 0.6).to(torch.uint8) if drop else None
    p = 0.4
    gp = torch.randn(M, Cn, generator=g) / M
    extra = torch.randn(M, H, generator=g) if ext else None
    gext = torch.randn(M, H, generator=g) if ext else None
    from ta3n_b200.functional import DropSpec
    ds = DropSpec(p, keep.to(_dev())) if drop else DropSpec()
    dc = ds.cstruct()
    dref = None if dc is None else C.byref(dc)
    xb, Wb, bb = Buf(M, H, init=x.to(_dev())), Buf(Cn, H, init=Wc.to(_dev())), Buf(Cn, init=bc.to(_dev()))
    dropped, pred = Buf(M, H), Buf(M, Cn)
    L.check(lib.ta3n_video_head_fwd(xb.p, M, H, Cn, Wb.p, bb.p, dref, dropped.p, pred.p, _st()))
    gpb = Buf(M, Cn, init=gp.to(_dev()))
    eb = None if extra is None else Buf(M, H, init=extra.to(_dev()))
    gxb = None if gext is None else Buf(M, H, init=gext.to(_dev()))
    dfv = None if no_dfeat else Buf(M, H)
    dWc, dbc = Buf(Cn, H), Buf(Cn)
    ws = _ws(lib.ta3n_video_head_bwd_workspace_bytes(M, H, Cn))
    L.check(lib.ta3n_video_head_bwd(dropped.p, M, H, Cn, Wb.p, dref, gpb.p, None if eb is None else eb.p,
                                    None if gxb is None else gxb.p, scale, None if dfv is None else dfv.p, dWc.p,
                                    dbc.p, ws.data_ptr(), ws.numel(), _st()))
    torch.cuda.synchronize()
    r64, r32 = _ref(_head_ref, x, Wc, bc, keep, p, gp, extra, gext, scale)
    check("dropped", dropped.t, r64["dropped"], r32["dropped"], dims=(0,))
    check("pred", pred.t, r64["pred"], r32["pred"], dims=(0,))
    if dfv is not None:
        check("d_feat_video", dfv.t, r64["d_feat_video"], r32["d_feat_video"], dims=(0,))
    check("dWc", dWc.t, r64["dWc"], r32["dWc"], dims=(0,))
    check("dbc", dbc.t, r64["dbc"], r32["dbc"], scale=r64["scale_dbc"])
    _guards(dropped, pred, dfv, dWc, dbc)


# ---- TRN at the documented limit: T = 33, R = 32 scales, 94 relations ---------------------------------------------
def _sampled_relations(T, seed):
    """The relation table shape of TRNmodule.py:30-41 (scale T: one relation, every smaller scale: three) with frame
    tuples drawn at random: enumerating the combinations is impossible at T = 33."""
    rng = random.Random(seed)
    tuples = [[tuple(range(T))]]
    for s in range(T - 1, 1, -1):
        tuples.append([tuple(sorted(rng.sample(range(T), s))) for _ in range(3)])
    return tuples


def _ctable(T, tuples):
    from ta3n_b200._lib import RelationTable
    R = len(tuples)
    keep = ((C.c_int * R)(*[len(r[0]) for r in tuples]), (C.c_int * R)(*[len(r) for r in tuples]))
    flat = [f for r in tuples for t in r for f in t]
    keep = keep + ((C.c_int * len(flat))(*flat),)
    return RelationTable(T, R, *keep), keep


def _trn_ref(dt, x, Ws, bs, tuples, gates, G, dx0):
    xx = _leaf(x, dt)
    w, b = [_leaf(t, dt) for t in Ws], [_leaf(t, dt) for t in bs]
    M = x.shape[0]
    acts, per_scale, q = [], [], 0
    for i, rels in enumerate(tuples):
        acc = 0
        for tau in rels:
            a = orc._relu(F.linear(F.relu(xx[:, list(tau), :].reshape(M, -1)), w[i], b[i]), gates[q])
            acts.append(a)
            acc = acc + a
            q += 1
        per_scale.append(acc)
    fr = torch.stack(per_scale, 1)
    gr = _grads((fr * G.to(dt)).sum(), [xx, *w, *b])
    R = len(tuples)
    return dict(act=torch.stack(acts).detach(), feat_rel=fr.detach(),
                dx=gr[0] + (0 if dx0 is None else dx0.to(dt)), dW=gr[1:1 + R], db=gr[1 + R:])


@pytest.mark.parametrize("engine,accumulate_dx", [("fp32", 0), ("fp32", 1), ("tf32x3", 0), ("tf32", 1)])
def test_trn_at_documented_limit(engine, accumulate_dx):
    """ta3n_trn_fwd / _bwd at T = 33 with a sampled relation table (94 relations, F = 64): the frame data-gradient
    groups exceed 64 tensor maps.  The exact engine is held to the file's bound; tf32x3 and tf32 to the path's
    tolerances of tests/test_gpu_parity.py, on the activation pattern they realised."""
    import ta3n_b200
    from tests.test_gpu_parity import GRAD_TOL, NOISE_SCALE, TOL
    ta3n_b200.set_gemm_engine(engine)
    L, lib = _lib()
    T, M, Fd, H = 33, 16, 64, 256
    tuples = _sampled_relations(T, seed=33)
    assert sum(len(r) for r in tuples) == 94
    tab, _keep = _ctable(T, tuples)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(M, T, Fd, generator=g)
    Ws = [torch.randn(H, len(r[0]) * Fd, generator=g) / math.sqrt(len(r[0]) * Fd) for r in tuples]
    bs = [0.1 * torch.randn(H, generator=g) for _ in tuples]
    G = torch.randn(M, T - 1, H, generator=g)
    dx0 = torch.randn(M, T, Fd, generator=g) if accumulate_dx else None
    Wd, bd = [w.to(_dev()) for w in Ws], [b.to(_dev()) for b in bs]
    xb = Buf(M, T, Fd, init=x.to(_dev()))
    act, fr = Buf(94, M, H), Buf(M, T - 1, H)
    ptrs = lambda ts: _pa([t.data_ptr() for t in ts])    # noqa: E731
    L.check(lib.ta3n_trn_fwd(xb.p, M, Fd, H, C.byref(tab), ptrs(Wd), ptrs(bd), 1, act.p, fr.p, _st()))
    Gb = Buf(M, T - 1, H, init=G.to(_dev()))
    dW = [torch.full_like(w, float("nan")) for w in Wd]
    db = [torch.full_like(b, float("nan")) for b in bd]
    dx = Buf(M, T, Fd, init=None if dx0 is None else dx0.to(_dev()))
    ws = _ws(lib.ta3n_trn_bwd_workspace_bytes(M, Fd, H, C.byref(tab)))
    L.check(lib.ta3n_trn_bwd(xb.p, M, Fd, H, C.byref(tab), ptrs(Wd), 1, act.p, Gb.p, ptrs(dW), ptrs(db), dx.p,
                             accumulate_dx, ws.data_ptr(), ws.numel(), _st()))
    torch.cuda.synchronize()
    gates = [a > 0 for a in act.cpu()]
    r64, r32 = _ref(_trn_ref, x, Ws, bs, tuples, gates, G, dx0)
    exact = engine == "fp32"
    tf, tg = (TOL_FP32, TOL_FP32) if exact else (TOL[engine], GRAD_TOL[engine])
    ns = 1.0 if exact else NOISE_SCALE[engine]
    check("act", act.t, r64["act"], r32["act"], dims=(0, 1) if exact else (), tol=tf, noise_scale=ns)
    check("feat_rel", fr.t, r64["feat_rel"], r32["feat_rel"], dims=(0, 1) if exact else (), tol=tf, noise_scale=ns)
    check("dx", dx.t, r64["dx"], r32["dx"], dims=(0, 1) if exact else (), tol=tg, noise_scale=ns)
    for i in range(T - 1):
        check(f"dW{i}", dW[i], r64["dW"][i], r32["dW"][i], tol=tg, noise_scale=ns)
        check(f"db{i}", db[i], r64["db"][i], r32["db"][i], tol=tg, noise_scale=ns)
    _guards(act, fr, dx)


# ================================================================================================
# 2. loss kernels, each term alone and at full weight
# ================================================================================================
def _loss_ref(dt, pv, labels, pr, pd, pf, Bs, vs, vt, gamma, flags):
    """main.py:446, 508-538, 559-562 on the real rows (source rows [0, vs), target rows [Bs, Bs + vt))."""
    v, r, d, f = (_leaf(t, dt) for t in (pv, pr, pd, pf))
    real = torch.cat([torch.arange(vs), torch.arange(Bs, Bs + vt)])
    loss = torch.zeros((), dtype=dt)
    if vs > 0:
        loss = loss + F.cross_entropy(v[:vs], labels[:vs])

    def dom_ce(t):                                       # t [M, k, 2]: mean over the real rows' k predictions
        k = t.shape[1]
        y = torch.cat([torch.zeros(vs * k, dtype=torch.long), torch.ones(vt * k, dtype=torch.long)])
        return F.cross_entropy(t[real].reshape(-1, 2), y)

    if vs + vt > 0:
        if flags & 1:
            loss = loss + dom_ce(r)
        if flags & 2:
            loss = loss + dom_ce(d.unsqueeze(1))
        if flags & 4:
            loss = loss + dom_ce(f)
        if flags & 8:
            loss = loss + gamma * orc.attentive_entropy(v[real], d[real])
    gv, gr, gd, gf = _grads(loss, [v, r, d, f], allow_unused=True)
    z = lambda g, t: torch.zeros_like(t) if g is None else g   # noqa: E731
    return dict(loss=loss.detach(), g_video=z(gv, v), g_rel=z(gr, r), g_dom=z(gd, d), g_frame=z(gf, f))


def _run_loss(Bs, Bt, R, T, Cn, gamma, flags, valid, saturate, seed):
    L, lib = _lib()
    M = Bs + Bt
    g = torch.Generator().manual_seed(seed)
    s = 40.0 if saturate else 1.0
    pv = torch.randn(M, Cn, generator=g) * (s if saturate else 2.0)
    pr, pd, pf = (torch.randn(M, *sh, generator=g) * s for sh in ((R, 2), (2,), (T, 2)))
    if saturate:                                         # |delta| of 30 to 80 on both sides of zero
        for t in (pr, pd, pf):
            t[..., 0] += torch.sign(t[..., 0]) * 30.0
        pv[:, 0] += 30.0
    labels = torch.randint(0, Cn, (Bs,), generator=g)
    vs, vt = (Bs, Bt) if valid is None else valid
    bufs = {k: Buf(*t.shape, init=t.to(_dev())) for k, t in (("pv", pv), ("pr", pr), ("pd", pd), ("pf", pf))}
    lab = labels.to(_dev())
    vr = None if valid is None else torch.tensor(valid, dtype=torch.int32, device=_dev())
    loss, gv, gr, gd, gf = Buf(1), Buf(M, Cn), Buf(M, R, 2), Buf(M, 2), Buf(M, T, 2)
    ws = _ws(lib.ta3n_loss_workspace_bytes(M))
    L.check(lib.ta3n_loss_fwd_bwd(bufs["pv"].p, lab.data_ptr(), bufs["pr"].p, bufs["pd"].p, bufs["pf"].p, Bs, Bt, T, R,
                                  Cn, gamma, flags, None if vr is None else vr.data_ptr(), loss.p, gv.p, gr.p, gd.p,
                                  gf.p, ws.data_ptr(), ws.numel(), _st()))
    torch.cuda.synchronize()
    r64, r32 = _ref(_loss_ref, pv, labels, pr, pd, pf, Bs, vs, vt, gamma, flags)
    check("loss", loss.t[0], r64["loss"], r32["loss"])
    check("g_pred_video", gv.t, r64["g_video"], r32["g_video"], dims=(0,))
    check("g_pred_rel", gr.t, r64["g_rel"], r32["g_rel"], dims=(0, 1))
    check("g_pred_dom_video", gd.t, r64["g_dom"], r32["g_dom"], dims=(0,))
    check("g_pred_frame", gf.t, r64["g_frame"], r32["g_frame"], dims=(0, 1))
    pad = torch.ones(M, dtype=torch.bool)
    pad[:vs] = False
    pad[Bs:Bs + vt] = False
    for name, b in (("video", gv), ("rel", gr), ("dom", gd), ("frame", gf)):
        assert bool((b.cpu()[pad] == 0).all()), f"padded rows of g_pred_{name} must be exactly zero"
    _guards(loss, gv, gr, gd, gf)


@pytest.mark.parametrize("gamma", [0.003, 1.0])
@pytest.mark.parametrize("flags", [1, 2, 4, 8, 15])
def test_loss_terms_alone_and_together(flags, gamma):
    """ta3n_loss_fwd_bwd with each term alone (relation / video / frame adversarial CE, attentive entropy) and all
    together, the entropy at the shipped gamma and at full weight; Bs != Bt, so a mean over the wrong rows shows."""
    _run_loss(13, 9, 4, 5, 12, gamma, flags, None, False, seed=flags * 10 + int(gamma))


@pytest.mark.parametrize("valid", [None, "short", "no_target"])
@pytest.mark.parametrize("Bs,Bt,R,T,Cn", [(7, 3, 1, 1, 2), (40, 25, 32, 33, 33), (5, 9, 4, 5, 1000),
                                          (300, 200, 4, 5, 12)])
def test_loss_shapes_and_padding(Bs, Bt, R, T, Cn, valid):
    """R in {1, 4, 32}, T in {1, 5, 33}, C in {2, 12, 33, 1000}; valid_rows absent, short on both sides, and with no
    real target row.  Padded rows must get exactly zero gradient."""
    v = {None: None, "short": (max(Bs - 2, 1), max(Bt - 1, 0)), "no_target": (Bs - 1, 0)}[valid]
    _run_loss(Bs, Bt, R, T, Cn, 1.0, 15, v, False, seed=Bs + Cn)


@pytest.mark.parametrize("gamma", [0.003, 1.0])
def test_loss_saturated_logits(gamma):
    """Domain and class logits saturated (|delta| of 30 to 80): softmax probabilities of e^-80 and entropies near 0."""
    _run_loss(17, 11, 4, 5, 12, gamma, 15, (15, 10), True, seed=5)


def _ce_ref(dt, pred, labels, vs, L0):
    p = _leaf(pred, dt)
    loss = torch.tensor(L0, dtype=dt) + (F.cross_entropy(p[:vs], labels[:vs]) if vs > 0 else 0)
    (g,) = _grads(loss, [p]) if vs > 0 else (torch.zeros_like(p),)
    return dict(loss=loss.detach(), g=g)


@pytest.mark.parametrize("rows,valid", [(0, None), (37, None), (37, 30), (37, 0)])
def test_ce_loss(rows, valid):
    """ta3n_ce_loss_fwd_bwd adds to *loss; rows = 0 is a no-op; short valid_rows (also zero real rows)."""
    L, lib = _lib()
    Cn = 33
    g = torch.Generator().manual_seed(rows + 1)
    pred = torch.randn(max(rows, 1), Cn, generator=g)[:rows] * 3
    labels = torch.randint(0, Cn, (rows,), generator=g)
    L0 = 0.625
    pb, lab = Buf(rows, Cn, init=pred.to(_dev())), labels.to(_dev())
    loss, gp = Buf(1, init=torch.full((1,), L0, device=_dev())), Buf(rows, Cn)
    vr = None if valid is None else torch.tensor([valid, 0], dtype=torch.int32, device=_dev())
    L.check(lib.ta3n_ce_loss_fwd_bwd(pb.p, lab.data_ptr(), rows, Cn, None if vr is None else vr.data_ptr(), loss.p,
                                     gp.p, _st()))
    torch.cuda.synchronize()
    if rows == 0:
        assert float(loss.cpu()[0]) == L0
        _guards(loss, gp)
        return
    vs = rows if valid is None else valid
    r64, r32 = _ref(_ce_ref, pred, labels, vs, L0)
    check("loss", loss.t[0], r64["loss"], r32["loss"])
    check("g_pred", gp.t, r64["g"], r32["g"], dims=(0,))
    assert bool((gp.cpu()[vs:] == 0).all())
    _guards(loss, gp)


def _mcd_ref(dt, p1, p2, vt, L0, GM):
    a, b = _leaf(p1, dt), _leaf(p2, dt)
    loss = torch.tensor(L0, dtype=dt)
    if vt > 0:
        loss = loss - orc.dis_MCD(a[:vt], b[:vt])
        g1, g2 = _grads(loss, [a, b])
    else:
        g1, g2 = torch.zeros_like(a), torch.zeros_like(b)
    return dict(loss=loss.detach(), g1=g1 + (0 if GM is None else GM.to(dt)), g2=g2)


@pytest.mark.parametrize("move", [True, False])
@pytest.mark.parametrize("rows,Cn,valid", [(45, 12, None), (45, 12, 40), (20, 1000, 17), (30, 7, 0)])
def test_mcd_loss(rows, Cn, valid, move):
    """ta3n_mcd_loss_fwd_bwd: g_move1 is added to g_pred1 and zeroed, on padded rows too; rows where pred1 == pred2
    have zero gradient (sign(0) = 0); no real target row adds 0 to the loss."""
    L, lib = _lib()
    g = torch.Generator().manual_seed(rows + Cn)
    p1 = torch.randn(rows, Cn, generator=g) * 2
    p2 = torch.randn(rows, Cn, generator=g) * 2
    p2[::5] = p1[::5]                                    # identical rows
    GM = torch.randn(rows, Cn, generator=g) if move else None
    L0 = 1.25
    b1, b2 = Buf(rows, Cn, init=p1.to(_dev())), Buf(rows, Cn, init=p2.to(_dev()))
    loss, g1, g2 = Buf(1, init=torch.full((1,), L0, device=_dev())), Buf(rows, Cn), Buf(rows, Cn)
    gm = None if GM is None else Buf(rows, Cn, init=GM.to(_dev()))
    vr = None if valid is None else torch.tensor([0, valid], dtype=torch.int32, device=_dev())
    L.check(lib.ta3n_mcd_loss_fwd_bwd(b1.p, b2.p, rows, Cn, None if vr is None else vr.data_ptr(), loss.p, g1.p, g2.p,
                                      None if gm is None else gm.p, _st()))
    torch.cuda.synchronize()
    vt = rows if valid is None else valid
    r64, r32 = _ref(_mcd_ref, p1, p2, vt, L0, GM)
    check("loss", loss.t[0], r64["loss"], r32["loss"], scale=torch.tensor(L0 + 1.0))
    check("g_pred1", g1.t, r64["g1"], r32["g1"], dims=(0,))
    check("g_pred2", g2.t, r64["g2"], r32["g2"], dims=(0,))
    same = torch.zeros(rows, dtype=torch.bool)
    same[::5] = True
    assert bool((g2.cpu()[same] == 0).all()), "rows with pred1 == pred2 must have zero gradient"
    assert bool((g2.cpu()[vt:] == 0).all())
    if gm is not None:
        assert bool((gm.cpu() == 0).all()), "g_move1 must be cleared"
        assert torch.equal(g1.cpu()[same | (torch.arange(rows) >= vt)], GM[same | (torch.arange(rows) >= vt)])
    else:
        assert bool((g1.cpu()[same] == 0).all())
    _guards(loss, g1, g2, gm)


# ================================================================================================
# 3. the whole step at fp32 grade, with the entropy term visible
# ================================================================================================
STEP_CASES = {
    # id: (mode, T, use_attn, use_attn_frame, class / domain weights, MCD mu or None)
    "legacy_t3": ("legacy", 3, "TransAttn", "none", False, None),
    "legacy_t5": ("legacy", 5, "TransAttn", "none", False, None),
    "legacy_t10": ("legacy", 10, "TransAttn", "none", False, None),
    "phased_t3": ("phased", 3, "TransAttn", "none", False, None),
    "phased_t5": ("phased", 5, "TransAttn", "none", False, None),
    "phased_t10": ("phased", 10, "TransAttn", "none", False, None),
    "legacy_t5_noattn": ("legacy", 5, "none", "none", False, None),
    "phased_t10_noattn": ("phased", 10, "none", "none", False, None),
    "legacy_t4_frameattn": ("legacy", 4, "TransAttn", "TransAttn", False, None),
    "phased_t5_weights": ("phased", 5, "TransAttn", "none", True, None),
    "mcd_t5_mu0": ("legacy", 5, "TransAttn", "none", False, 0.0),
    "mcd_t4_mu07": ("legacy", 4, "TransAttn", "none", False, 0.7),
}
BETA = (0.75, 0.6, 0.5)


def _step_inputs(T, use_attn, attn_frame, mcd_mu, seed):
    bs, bt, Cn = 13, 9, 12
    cfg = orc.PathConfig(num_class=Cn, num_segments=T, fc_dim=256, dropout_i=0.0, dropout_v=0.0, use_attn=use_attn,
                         use_attn_frame=attn_frame, ens_DA="none" if mcd_mu is None else "MCD")
    params = orc.init_params(cfg, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    for k in params:                                     # trained-like weights: logits of O(1)
        if params[k].dtype.is_floating_point and "weight" in k and \
                (k.startswith(orc.USED_PARAM_PREFIXES) or k.startswith("fc_classifier_video_source_2")):
            params[k] = params[k] + 0.02 * torch.randn(params[k].shape, generator=g)
    xs = torch.randn(bs, T, orc.FEATURE_DIM, generator=g)
    xt = torch.randn(bt, T, orc.FEATURE_DIM, generator=g) + 0.2
    labels = torch.randint(0, Cn, (bs,), generator=g)
    return cfg, params, xs, xt, labels


def _pool_gates(pool, rows_f, rows_v, frame_disc=True, video_disc=True):
    g = {"shared": rows_f(pool["feat"]) > 0, "trn": [rows_v(a) > 0 for a in pool["act"]],
         "rel_disc": [rows_v(h) > 0 for h in pool["hid_r"]]}
    if frame_disc:
        g["frame_disc"] = rows_f(pool["hid_f"]) > 0
    if video_disc:
        g["video_disc"] = rows_v(pool["hid_v"]) > 0
    return g


def _check_grads(named, g64, g32):
    for name, go in g64.items():
        assert named[name].grad is not None, name
        dims = (0,) if name.startswith("fc_classifier_video_source") and name.endswith("weight") else ()
        check(f"grad {name}", named[name].grad, go, g32[name], dims=dims)


@pytest.mark.parametrize("gamma", [1.0, 0.003])
@pytest.mark.parametrize("case", list(STEP_CASES))
def test_train_step_at_fp32_grade(case, gamma):
    """TrainStep under the exact engine, dropout off, against the fp64 oracle on the ReLU pattern the step realised:
    the loss and every parameter gradient under the file's bound.  Both executors; T = 3, 5, 10 (R = 2, 4, 9: the
    step program's relation rows take the scales in rounds of four and then two, R = 2 and 9 end in a partial round,
    R = 9 also passes the 8 warps of the relation kernels); TransAttn and none; frame attention; class and domain
    weights; MCD with mu 0 and 0.7.  At gamma = 1 the attentive entropy carries as much weight as the class loss."""
    from tests.test_gpu_parity import build_model
    from ta3n_b200.train import TrainStep
    mode, T, ua, uaf, weights, mu = STEP_CASES[case]
    cfg, params, xs, xt, labels = _step_inputs(T, ua, uaf, mu, seed=T * 7 + len(case))
    bs, bt, Cn = xs.shape[0], xt.shape[0], cfg.num_class
    cw = dw = None
    kw = {}
    if weights:
        cw = torch.rand(Cn, generator=torch.Generator().manual_seed(2)) + 0.25
        dw = (0.6, 1.7)
        kw = dict(class_weight=cw, domain_weight=dw)
    if mu is not None:
        kw["mu"] = mu
    model = build_model(cfg, params, train=True)
    step = TrainStep(model, bs, bt, BETA, gamma=gamma, use_graph=False, mode=mode, **kw)
    loss = step(xs, xt, labels)
    torch.cuda.synchronize()
    p64 = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in params.items()}
    cpu = lambda t: t.cpu()                              # noqa: E731
    gates = _pool_gates(step.bufs.pool, cpu, cpu)
    if mu is None:
        l64, _, g64 = orc.train_step(p64, xs.double(), xt.double(), labels, BETA, cfg, gamma, train=True, gates=gates,
                                     class_weight=None if cw is None else cw.double(),
                                     domain_weight=None if dw is None else torch.tensor(dw).double())
        l32, _, g32 = orc.train_step(params, xs, xt, labels, BETA, cfg, gamma, train=True, gates=gates,
                                     class_weight=cw, domain_weight=None if dw is None else torch.tensor(dw))
    else:
        T_ = cfg.num_segments
        g2 = _pool_gates(step.bufs2.pool, lambda t: t[:bt * T_].cpu(), lambda t: t[:bt].cpu(),
                         frame_disc=cfg.use_attn_frame != "none", video_disc=False)
        _, gt2 = orc.split_gates(g2, 0, T_)
        l64, _, _, g64 = mcd.mcd_train_step(p64, xs.double(), xt.double(), labels, BETA, mu, cfg, gamma, gates=gates,
                                            gates2=gt2)
        l32, _, _, g32 = mcd.mcd_train_step(params, xs, xt, labels, BETA, mu, cfg, gamma, gates=gates, gates2=gt2)
    check("loss", loss.cpu()[0], l64, l32)
    _check_grads(dict(model.named_parameters()), {k: v for k, v in g64.items() if v is not None}, g32)


def _variant_oracle(cfg, params, xs, xt, labels, dtype, gamma):
    p = {k: (v.to(dtype).requires_grad_(True) if v.dtype.is_floating_point else v) for k, v in params.items()}
    o = orc.forward(p, xs.to(dtype), xt.to(dtype), BETA, 0.0, cfg, train=True, reverse=False)
    loss = orc.compose_loss(o, labels, gamma, use_attn=cfg.use_attn)
    loss.backward()
    return loss.detach(), {k: v.grad for k, v in p.items() if v.dtype.is_floating_point and v.grad is not None}


@pytest.mark.parametrize("gamma", [1.0, 0.003])
@pytest.mark.parametrize("variant", ["general", "avgpool"])
def test_video_model_variant_at_fp32_grade(variant, gamma):
    """One autograd VideoModel step each for use_attn='general' and frame_aggregation='avgpool' (TransAttn), loss and
    every parameter gradient under the file's bound."""
    from tests.test_gpu_parity import build_model
    from ta3n_b200.loss import ta3n_loss
    T, Cn = 5, 9
    if variant == "general":
        cfg = orc.PathConfig(num_class=Cn, num_segments=T, fc_dim=256, dropout_i=0.0, dropout_v=0.0, use_attn="general")
    else:
        cfg = orc.PathConfig(num_class=Cn, num_segments=T, fc_dim=256, dropout_i=0.0, dropout_v=0.0,
                             use_attn="TransAttn", frame_aggregation="avgpool")
    params = orc.init_params(cfg, seed=61)
    g = torch.Generator().manual_seed(62)
    for k in params:
        if params[k].dtype.is_floating_point and k.startswith(orc.USED_PARAM_PREFIXES) and "weight" in k:
            params[k] = params[k] + 0.02 * torch.randn(params[k].shape, generator=g)
    xs = torch.randn(11, T, orc.FEATURE_DIM, generator=g)
    xt = torch.randn(8, T, orc.FEATURE_DIM, generator=g) + 0.3
    labels = torch.randint(0, Cn, (11,), generator=g)
    l64, g64 = _variant_oracle(cfg, params, xs, xt, labels, torch.float64, gamma)
    l32, g32 = _variant_oracle(cfg, params, xs, xt, labels, torch.float32, gamma)
    model = build_model(cfg, params, train=True)
    outs = model(xs.to(_dev()), xt.to(_dev()), list(BETA), 0.0, is_train=True, reverse=False)
    loss = ta3n_loss(outs, labels.to(_dev()), gamma, use_attn=cfg.use_attn)
    loss.backward()
    torch.cuda.synchronize()
    check("loss", loss.detach().cpu(), l64, l32)
    named = dict(model.named_parameters())
    for name, go in g64.items():
        if name == "attn_layer.2.bias":                  # zero by construction (softmax shift invariance)
            assert float(named[name].grad.norm()) <= 1e-5 * max(1.0, float(named["attn_layer.2.weight"].grad.norm()))
            continue
        dims = (0,) if name == "fc_classifier_video_source.weight" else ()
        check(f"grad {name}", named[name].grad, go, g32[name], dims=dims)
