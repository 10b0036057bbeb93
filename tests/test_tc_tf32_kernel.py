"""The plain tensor-core kernel (seg_gemm_tc_kernel<A_KMAJ, B_KMAJ>) and every backward GEMM, per tile against fp64.

Under the default engine (tf32x3) this kernel runs every data-gradient and every weight-gradient GEMM of the step
except the small weight gradients; under set_gemm_engine('tf32') it runs everything.  Two bounds:

  Tier E (exact operands, any route: plain, precise or SIMT).  Every GEMM operand is tf32-representable (its low 13
         mantissa bits are zero), so every rounding rule the tensor maps or the tensor core could apply is the
         identity and the products are exact: only fp32 accumulation remains.
             ||C - R|| <= 2e-5 ||R||   per tensor, per slice (frame of dx, (scale, slot) slab of a TRN dW,
                                       relation) and per 128 x 128 tile (with the tile-norm floor of _check_tiles)
         Operands that a row kernel forms from several inputs (dpre, the discriminator's dH, the TRN's dz, dHid with
         use_attn 0 / 2) are exact because their inputs lie on a coarse grid (k 2^-e, |k| < 32) and the dropout
         scales and beta are powers of two or short; each test asserts that on its fp64 restatement before it trusts
         the bound.  The inputs hold exact zeros, so the ReLU masks and EPI_GATE see ties at 0.
  Tier R (raw randn fp32 operands, plain kernel).  The TFLOAT32 tensor maps round each operand to nearest while
         filling shared memory (gemm_wgmma.cuh: encode_map), so a product is off by ~3e-4 normwise and unbiased:
             normwise <= 5e-4, per tile <= 6e-4, signed bias |sum((C - R) R) / sum(R^2)| <= 5e-5
         on mixed-sign and on all-positive operands.  Truncating raw fp32 words instead gives a bias of about -7e-4.
         The small weight gradients that run on the precise kernel under tf32x3 are held to 2e-5 there.

Every case asserts the GEMM kernels it launched (torch.profiler names, launch counts, split-K reduces) against a
restatement of the dispatcher (run_gemm, tc_group_ok, plan_splitk, launch_tc), writes into NaN-filled outputs behind
sentinel guards (EPI_ACCUM outputs pre-filled with known values), and reruns bit-identically.
"""
import ctypes as C
import math
import re
from collections import Counter

import pytest
import torch

from tests.test_rowops_fp32 import Buf, _ctable, _sampled_relations, check
from tests.test_x3_kernel import _check_tiles, _kernels, _Out

pytestmark = pytest.mark.gpu

TIER_E = 2e-5
TIER_R, TIER_R_TILE, TIER_R_BIAS = 5e-4, 6e-4, 5e-5
PAD_VALUE = 1024.0           # between the rows of padded operands: a read of it would show as a huge error
MAX_GROUPS, MAX_SEGS, MAX_MAPS = 48, 128, 64
SMALL_MN, SMALL_FLOP = 256 * 256, 3e8
_WORST = []

__all__ = ["tf32_exact", "is_tf32", "grid"]


# ------------------------------------------------------------------------------------------------
# operands (host-only helpers; tests/test_tc_tf32_operands.py checks them without a GPU)
# ------------------------------------------------------------------------------------------------
def tf32_exact(t):
    """t as fp32 with the low 13 mantissa bits cleared: a tf32 value, which every rounding rule leaves unchanged."""
    t = t.detach().to(torch.float32).contiguous()
    return (t.view(torch.int32) & ~0x1FFF).view(torch.float32)


def is_tf32(t):
    """Every entry of t (any float dtype) is exactly an fp32 value whose low 13 mantissa bits are zero."""
    t = t.detach()
    f = t.to(torch.float32)
    if not torch.equal(f.to(t.dtype), t):
        return False
    return bool(((f.contiguous().view(torch.int32) & 0x1FFF) == 0).all())


def grid(shape, e, g, relu=False):
    """Integers k in [-31, 31] times 2^-e (exact zeros included): sums of a few products of such values stay
    tf32-representable.  relu: the negative ones set to zero (a ReLU pattern with many ties at 0)."""
    t = torch.randint(-31, 32, tuple(shape), generator=g).to(torch.float32) * 2.0 ** -e
    return t.clamp_min(0.0) if relu else t


def _assert_tf32(what, *ts):
    for i, t in enumerate(ts):
        assert is_tf32(t), f"{what}: GEMM operand {i} of the fp64 restatement is not tf32-representable"


# ------------------------------------------------------------------------------------------------
# bounds
# ------------------------------------------------------------------------------------------------
def _dev():
    return torch.device("cuda:0")


def _st():
    return torch.cuda.current_stream().cuda_stream


def _lib():
    from ta3n_b200 import _lib as L
    return L, L.load()


def _pa(ptrs):
    from ta3n_b200._lib import ptr_array
    return ptr_array(ptrs)


def _engine(name):
    import ta3n_b200
    ta3n_b200.set_gemm_engine(name)


@pytest.fixture(autouse=True)
def _restore_engine(request):
    _WORST.clear()
    yield
    _engine("tf32x3")
    if _WORST:
        print(f"\n[tc-tf32] {request.node.name}: worst error/bound {max(_WORST):.3f}")


def _mm64(a, b):
    """a @ b in fp64, computed on the GPU from 1 GFLOP on (as test_x3_kernel._mm), returned on the GPU."""
    big = 2.0 * a.shape[0] * a.shape[1] * b.shape[1] >= 1e9
    d = _dev() if big else torch.device("cpu")
    return (a.to(d, torch.float64) @ b.to(d, torch.float64)).to(_dev())


def _planes(t):
    t = t.detach()
    return t.reshape(-1, *t.shape[-2:]) if t.dim() >= 2 else t.reshape(1, 1, -1)


def tier_e(what, got, ref, tol=TIER_E):
    """got against the fp64 ref [..., M, N] (a stack of GEMM outputs): per tensor, per plane and per tile."""
    got, ref = _planes(got), _planes(ref)
    worst = _check_tiles(what, got, ref, tol=tol)
    d = (got.to(_dev(), torch.float64) - ref.to(_dev(), torch.float64)).flatten(1).norm(dim=1)
    r = ref.to(_dev(), torch.float64).flatten(1).norm(dim=1)
    ratio = d / (tol * r).clamp_min(1e-300)
    i = int(ratio.argmax())
    assert float(ratio[i]) <= 1.0, f"{what}: plane {i} rel err {float(d[i] / r[i]):.2e} (bound {tol:.0e})"
    worst = max(worst, float(ratio.max()))
    _WORST.append(worst)
    return worst


def tier_r(what, got, ref):
    """Round to nearest, not truncation: normwise, per tile and the signed relative bias."""
    got, ref = _planes(got).to(_dev(), torch.float64), _planes(ref).to(_dev(), torch.float64)
    diff = got - ref
    err = (diff.norm() / ref.norm()).item()
    bias = ((diff * ref).sum() / (ref * ref).sum()).item()
    assert err <= TIER_R, f"{what}: normwise rel err {err:.2e} (bound {TIER_R:.0e})"
    assert abs(bias) <= TIER_R_BIAS, f"{what}: relative bias {bias:.2e} (bound {TIER_R_BIAS:.0e}; truncation: -7e-4)"
    worst = max(_check_tiles(what, got, ref, tol=TIER_R_TILE), err / TIER_R, abs(bias) / TIER_R_BIAS)
    print(f"[tc-tf32] {what}: normwise {err:.2e}, bias {bias:+.2e}")
    _WORST.append(worst)
    return worst


def _twice(run, outs):
    """run() (which pre-fills its outputs) under the profiler, then again: the outputs bit-identical."""
    names = _kernels(run)
    first = [o.clone() for o in outs]
    run()
    torch.cuda.synchronize()
    for i, (a, o) in enumerate(zip(first, outs)):
        assert torch.equal(a.nan_to_num(7.0), o.nan_to_num(7.0)), f"output {i}: a second run gave a different result"
    return names


# ------------------------------------------------------------------------------------------------
# which GEMM kernels a plan launches: a restatement of run_gemm / tc_group_ok / plan_splitk / launch_tc
# ------------------------------------------------------------------------------------------------
def _gemm_launches(names):
    c = Counter()
    for n in names:
        m = re.search(r"seg_gemm_(tc_x3|tc|simt)_kernel<(true|false),(true|false)>", n)
        if m:
            c[f"{ {'tc_x3': 'x3', 'tc': 'tc', 'simt': 'simt'}[m.group(1)]}<{m.group(2)},{m.group(3)}>"] += 1
        elif "splitk_reduce_v4_kernel" in n:
            c["reduce_v4"] += 1
        elif re.search(r"splitk_reduce_kernel\b", n):
            c["reduce"] += 1
    return c


class G:
    """One group of a plan: C[M, N] over segments (A key, B key, K length, both operands TMA-able)."""

    def __init__(self, M, N, vec_c=True):
        self.M, self.N, self.segs, self.vec_c = M, N, [], vec_c

    def seg(self, a, b, k, ok=True):
        self.segs.append((a, b, k, ok))
        return self

    @property
    def k(self):
        return sum(s[2] for s in self.segs)

    def keys(self):
        return {s[0] for s in self.segs} | {s[1] for s in self.segs}


def _aligned(ptr, ld):
    return ptr % 16 == 0 and ld % 4 == 0


def _splits(gs, bm, bn, bk, min_chunks):
    tiles = sum(math.ceil(g.M / bm) * math.ceil(g.N / bn) for g in gs)
    if 2 * tiles > 132:
        return [1] * len(gs)
    out = []
    for g in gs:
        ks = min(132 // tiles, sum(math.ceil(s[2] / bk) for s in g.segs) // min_chunks, 8)
        out.append(ks if ks >= 2 else 1)
    return out


def _pack(gs, maps):
    """Launches of launch_tc / launch_simt: lists of group indices of gs (already in launch order)."""
    launches, i = [], 0
    while i < len(gs):
        local, cur, ns = set(), [], 0
        while i < len(gs) and len(cur) < MAX_GROUPS:
            g = gs[i]
            if ns + len(g.segs) > MAX_SEGS:
                break
            if maps:
                fresh = g.keys() - local
                if len(local) + len(fresh) > MAX_MAPS:
                    break
                local |= fresh
            cur.append(i)
            ns += len(g.segs)
            i += 1
        launches.append(cur)
    return launches


def expect(gs, engine, a_kmaj, b_kmaj, relu_load=False, arena=False):
    """Counter of the GEMM kernels run_gemm launches for the plan gs (as _gemm_launches names them)."""
    lay = f"<{'true' if a_kmaj else 'false'},{'true' if b_kmaj else 'false'}>"
    c = Counter()
    fine, tc, simt = [], [], []
    for g in gs:
        ok = (not relu_load and g.M * g.N >= 64 * 64 and len(g.segs) <= MAX_SEGS and all(s[3] for s in g.segs)
              and len(g.keys()) <= MAX_MAPS)
        tiny = (engine == "tf32x3" and not a_kmaj and not b_kmaj and g.M * g.N <= SMALL_MN
                and 2.0 * g.M * g.N * g.k <= SMALL_FLOP)
        (simt if not ok else fine if tiny else tc).append(g)
    for kind, part, split in (("x3", fine, False), ("tc", tc, arena)):
        if not part:
            continue
        ks = _splits(part, 128, 128, 32, 4) if split else [1] * len(part)
        order = sorted(range(len(part)), key=lambda i: -(part[i].k // ks[i]))
        part, ks = [part[i] for i in order], [ks[i] for i in order]
        for launch in _pack(part, maps=True):
            c[kind + lay] += 1
            sp = [i for i in launch if ks[i] > 1]
            if sp:
                c["reduce_v4" if all(part[i].vec_c and part[i].N % 4 == 0 for i in sp) else "reduce"] += 1
    if simt:
        ks = _splits(simt, 64, 64, 16, 8) if arena else [1] * len(simt)
        for launch in _pack(simt, maps=False):
            c["simt" + lay] += 1
            if any(ks[i] > 1 for i in launch):
                c["reduce"] += 1
    return c


def _assert_routes(what, names, want, run, sessions=3):
    """The GEMM launches in names are want.  A profiler session now and then loses some of a run's kernel records;
    when the recorded launches are a strict subset of want, run() (idempotent) is profiled again, at most `sessions`
    times in all.  A launch beyond want fails at once."""
    got = _gemm_launches(names)
    for _ in range(sessions - 1):
        if got == want or any(got[k] > want[k] for k in got):
            break
        print(f"[tc-tf32] {what}: the profiler recorded {dict(got)} of {dict(want)}; profiling the run again")
        got = _gemm_launches(_kernels(run))
    assert got == want, f"{what}: GEMM launches {dict(got)}, expected {dict(want)}"


def _small_route(engine, M, N, K):
    return engine == "tf32x3" and M * N <= SMALL_MN and 2.0 * M * N * K <= SMALL_FLOP


# ------------------------------------------------------------------------------------------------
# A. ta3n_gemm_ex in all four operand layouts
# ------------------------------------------------------------------------------------------------
class _Mat:
    """A matrix [rows, cols] stored row-major with row pitch ld at float offset off of a fresh allocation; the
    padding between rows holds PAD_VALUE."""

    def __init__(self, m, ld, off):
        rows, cols = m.shape
        self.buf = torch.full((off + rows * ld + 64,), PAD_VALUE, device=_dev())
        self.buf[off:off + rows * ld].view(rows, ld)[:, :cols] = m.to(_dev())
        self.p = self.buf[off:].data_ptr()


class _COut:
    """C [M, N] with row pitch ldc at float offset off: NaN inside, SENTINEL in the padding and behind."""
    SENTINEL = -1234.5

    def __init__(self, M, N, ldc, off):
        self.buf = torch.full((off + M * ldc + 4096,), self.SENTINEL, device=_dev())
        self.view = self.buf[off:off + M * ldc].view(M, ldc)
        self.t = self.view[:, :N]
        self.mask = torch.ones_like(self.buf, dtype=torch.bool)
        self.mask[off:off + M * ldc].view(M, ldc)[:, :N] = False
        self.p = self.view.data_ptr()

    def reset(self):
        self.t.fill_(float("nan"))

    def check_guard(self, what):
        bad = int((self.buf[self.mask] != self.SENTINEL).sum())
        assert bad == 0, f"{what}: {bad} floats outside C were written"


def _gemm_ex_setup(A, B, a_kmaj, b_kmaj, pad, cpad, off):
    """Operands of C = A @ B (A [M, K], B [K, N]) placed as the layouts read them; returns the call and its plan."""
    M, K = A.shape
    N = B.shape[1]
    lda = (K if a_kmaj else M) + pad
    ldb = (K if b_kmaj else N) + pad
    ldc = N + cpad
    Am = _Mat(A if a_kmaj else A.t(), lda, off)
    Bm = _Mat(B.t() if b_kmaj else B, ldb, off)
    out = _COut(M, N, ldc, off)
    ok = _aligned(Am.p, lda) and _aligned(Bm.p, ldb)
    g = G(M, N, vec_c=ldc % 4 == 0 and out.p % 16 == 0).seg(("A", Am.p), ("B", Bm.p), K, ok)
    return Am, Bm, out, lda, ldb, ldc, g


def _gemm_ex_run(A, B, a_kmaj, b_kmaj, engine, pad=0, cpad=0, off=0, ws=False):
    L, lib = _lib()
    _engine(engine)
    M, K = A.shape
    N = B.shape[1]
    Am, Bm, out, lda, ldb, ldc, g = _gemm_ex_setup(A, B, a_kmaj, b_kmaj, pad, cpad, off)
    w = torch.empty(16 << 20, dtype=torch.uint8, device=_dev()) if ws else None

    def run():
        out.reset()
        L.check(lib.ta3n_gemm_ex(Am.p, lda, a_kmaj, Bm.p, ldb, b_kmaj, out.p, ldc, M, N, K,
                                 None if w is None else w.data_ptr(), 0 if w is None else w.numel(), _st()))

    names = _twice(run, [out.t])
    out.check_guard("gemm_ex")
    want = expect([g], engine, bool(a_kmaj), bool(b_kmaj), arena=ws)
    _assert_routes(f"gemm_ex {M}x{N}x{K} a_kmaj={a_kmaj} b_kmaj={b_kmaj}", names, want, run)
    return out.t, want


LAYOUTS = [(1, 1), (1, 0), (0, 0), (0, 1)]
# (id, M, N, K, pad of lda / ldb, pad of ldc, float offset of every base, split-K workspace)
GEMM_E = [
    ("mn128", 256, 384, 96, 0, 0, 0, False),            # MN multiples of 128, K three whole slabs
    ("mn32-k33-base16", 96, 160, 33, 0, 0, 4, False),   # rank-3 MN-major maps, partial tile; bases 16 B, not 128 B
    ("ragged-padded", 200, 136, 500, 8, 4, 0, False),   # four 2-D boxes per MN-major slab; padded leading dimensions
    ("below32", 24, 200, 20, 0, 0, 0, False),           # M and K below 32
    ("first-wave", 2048, 2176, 40, 0, 0, 0, False),     # 272 tiles: more than one per SM, the tile remap
    ("k5120", 512, 1024, 5120, 0, 0, 0, False),         # K of the cfg5 shared-layer weight gradient
    ("split-v4", 256, 256, 2048, 0, 0, 0, True),        # split K 8 ways, vectorised reduce
    ("split-scalar", 256, 256, 2048, 0, 1, 0, True),    # ldc 257: the scalar reduce
    ("simt-ld", 200, 136, 500, 1, 0, 0, False),         # ld % 4 != 0
    ("simt-base4", 96, 160, 300, 0, 0, 1, False),       # 4-byte aligned bases
    ("simt-small", 60, 60, 300, 0, 0, 0, False),        # M N < 4096
]


@pytest.mark.parametrize("engine", ["tf32", "tf32x3"])
@pytest.mark.parametrize("a_kmaj,b_kmaj", LAYOUTS, ids=[f"a{a}b{b}" for a, b in LAYOUTS])
@pytest.mark.parametrize("case", GEMM_E, ids=[c[0] for c in GEMM_E])
def test_gemm_ex_exact_operands(case, a_kmaj, b_kmaj, engine):
    """Tier E in every layout, map route, placement, split and fallback; under tf32x3 the small M-major x N-major
    products take the precise kernel, everything else routes as under tf32."""
    cid, M, N, K, pad, cpad, off, ws = case
    g = torch.Generator().manual_seed(M + 3 * N + 7 * K + 11 * a_kmaj + 13 * b_kmaj)
    A = tf32_exact(torch.randn(M, K, generator=g))
    B = tf32_exact(torch.randn(K, N, generator=g))
    A[torch.rand(M, K, generator=g) < 0.05] = 0.0
    _assert_tf32(cid, A, B)
    got, want = _gemm_ex_run(A, B, a_kmaj, b_kmaj, engine, pad, cpad, off, ws)
    tier_e(f"gemm_ex {cid} a{a_kmaj}b{b_kmaj} {engine} {dict(want)}", got, _mm64(A, B))


# (M, N, K): rank-3 maps for MN-major operands, and the 2-D boxes
GEMM_R = [(512, 512, 1024), (500, 300, 1000)]


@pytest.mark.parametrize("a_kmaj,b_kmaj", LAYOUTS, ids=[f"a{a}b{b}" for a, b in LAYOUTS])
@pytest.mark.parametrize("M,N,K", GEMM_R)
def test_gemm_ex_raw_operands_round_to_nearest(M, N, K, a_kmaj, b_kmaj):
    """Tier R on raw randn operands (mixed sign) and on all-positive ones, plain kernel."""
    g = torch.Generator().manual_seed(M + N + K + a_kmaj + 2 * b_kmaj)
    for sign in ("mixed", "positive"):
        A, B = torch.randn(M, K, generator=g), torch.randn(K, N, generator=g)
        if sign == "positive":
            A, B = A.abs(), B.abs()
        got, want = _gemm_ex_run(A, B, a_kmaj, b_kmaj, "tf32")
        assert set(want) == {f"tc<{'true' if a_kmaj else 'false'},{'true' if b_kmaj else 'false'}>"}, want
        tier_r(f"gemm_ex raw {sign} {M}x{N}x{K} a{a_kmaj}b{b_kmaj}", got, _mm64(A, B))


@pytest.mark.parametrize("M,N,K", [(256, 256, 1024), (200, 136, 2000)])
def test_small_weight_gradient_is_precise_on_raw_operands(M, N, K):
    """Under tf32x3 an M-major x N-major product with M N <= 256^2 and <= 0.3 GFLOP runs on the precise kernel."""
    g = torch.Generator().manual_seed(M * N + K)
    A, B = torch.randn(M, K, generator=g), torch.randn(K, N, generator=g)
    got, want = _gemm_ex_run(A, B, 0, 0, "tf32x3", ws=True)
    assert want == Counter({"x3<false,false>": 1}), want
    tier_e(f"gemm_ex raw small {M}x{N}x{K} tf32x3", got, _mm64(A, B))


def test_map_cache_keeps_raw_and_rounded_maps_apart():
    """The same pointers and shapes, alternately through the precise kernel (FLOAT32 maps: raw words) and the plain
    one (TFLOAT32 maps: rounded by the TMA).  The plain result stays unbiased and identical each time: MapKey.raw
    keeps the two cached maps apart."""
    L, lib = _lib()
    M, N, K = 256, 256, 1024
    g = torch.Generator().manual_seed(5)
    A, B = torch.randn(M, K, generator=g).abs(), torch.randn(K, N, generator=g).abs()
    ref = _mm64(A, B)
    At, Bn = A.t().contiguous().to(_dev()), B.contiguous().to(_dev())
    Cx, Cp = torch.empty(M, N, device=_dev()), torch.empty(M, N, device=_dev())
    plain = []
    for _ in range(2):
        for engine, out in (("tf32x3", Cx), ("tf32", Cp)):
            _engine(engine)
            out.fill_(float("nan"))
            run = lambda: L.check(lib.ta3n_gemm_ex(At.data_ptr(), M, 0, Bn.data_ptr(), N, 0, out.data_ptr(), N,  # noqa
                                                   M, N, K, None, 0, _st()))
            names = _kernels(run)
            kind = "x3" if engine == "tf32x3" else "tc"
            _assert_routes(engine, names, Counter({kind + "<false,false>": 1}), run)
            if engine == "tf32x3":
                tier_e("cache: precise", Cx, ref)
            else:
                tier_r("cache: plain", Cp, ref)
                plain.append(Cp.clone())
    assert torch.equal(plain[0], plain[1])


# ------------------------------------------------------------------------------------------------
# B. backward entry points on exact operands
# ------------------------------------------------------------------------------------------------
def _ws(nbytes):
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=_dev())


def _ref_dev(t):
    return t.to(_dev(), torch.float64)


# ---- shared layer: dW [F, D] = dpre^T x over the source and the target rows ----------------------------------------
def _shared_inputs(rows_s, rows_t, D, F, p, ext, g):
    x = tf32_exact(torch.randn(rows_s + rows_t, D, generator=g))
    x[torch.rand(x.shape, generator=g) < 0.02] = 0.0
    feat = grid((rows_s + rows_t, F), 4, g, relu=True)
    dfeat = grid((rows_s + rows_t, F), 6, g)
    gext = grid((rows_s + rows_t, F), 6, g) if ext else None
    scale = 1.0 / (1.0 - p)
    dpre = (_ref_dev(dfeat) + (0 if gext is None else _ref_dev(gext))) * (_ref_dev(feat) > 0) * scale
    return x, feat, dfeat, gext, dpre


def _shared_call(lib, xs, rows_s, xt, rows_t, D, F, feat, dfeat, gext, p, dW, db, ws):
    return lib.ta3n_shared_fc_bwd(xs.data_ptr(), rows_s, None if xt is None else xt.data_ptr(), rows_t, D, F,
                                  feat.data_ptr(), dfeat.data_ptr(), None if gext is None else gext.data_ptr(), p,
                                  dW.ptr(), db.ptr(), ws.data_ptr(), ws.numel(), _st())


def _shared_plan(F, D, rows_s, rows_t, xs, xt):
    gr = G(F, D)
    if rows_s:
        gr.seg(("dpre", 0), ("x", xs.data_ptr()), rows_s)
    if rows_t:
        gr.seg(("dpre", rows_s), ("x", xt.data_ptr()), rows_t)
    return gr


SHARED = [(512, 1001, 1503, 0.5, True), (1024, 777, 0, 0.0, False), (512, 2560, 2560, 0.0, True),
          (1024, 2531, 2589, 0.5, False)]


@pytest.mark.parametrize("engine", ["tf32", "tf32x3"])
@pytest.mark.parametrize("F,rows_s,rows_t,p,ext", SHARED, ids=[f"F{c[0]}-{c[1]}+{c[2]}-p{c[3]}-ext{int(c[4])}"
                                                                for c in SHARED])
def test_shared_fc_bwd(F, rows_s, rows_t, p, ext, engine):
    """ta3n_shared_fc_bwd at D = 2048: ragged source / target segments (K not a multiple of 32), dropout p = 0 and
    0.5, g_feat_ext, up to 5120 rows (the cfg5 shape)."""
    L, lib = _lib()
    _engine(engine)
    D = 2048
    g = torch.Generator().manual_seed(F + rows_s + rows_t)
    x, feat, dfeat, gext, dpre = _shared_inputs(rows_s, rows_t, D, F, p, ext, g)
    _assert_tf32("shared dpre / x", dpre, x)
    d = _dev()
    xs, xt = x[:rows_s].contiguous().to(d), (x[rows_s:].contiguous().to(d) if rows_t else None)
    dfeat_d, feat_d, gext_d = dfeat.to(d), feat.to(d), None if gext is None else gext.to(d)
    dfb = torch.empty_like(dfeat_d)
    dW, db = _Out(F, D), _Out(F)
    ws = _ws(lib.ta3n_shared_fc_bwd_workspace_bytes(rows_s + rows_t, D, F))

    def run():
        dfb.copy_(dfeat_d)
        dW.t.fill_(float("nan"))
        db.t.fill_(float("nan"))
        L.check(_shared_call(lib, xs, rows_s, xt, rows_t, D, F, feat_d, dfb, gext_d, p, dW, db, ws))

    names = _twice(run, [dW.t, db.t, dfb])
    dW.check_guard("dW")
    db.check_guard("db")
    want = expect([_shared_plan(F, D, rows_s, rows_t, xs, xt)], engine, False, False, arena=True)
    _assert_routes("shared_fc_bwd", names, want, run)
    assert torch.equal(dfb.double(), dpre), "dpre (written into dfeat) is not exact"
    tier_e(f"shared dW F={F} rows={rows_s}+{rows_t} p={p} {engine} {dict(want)}", dW.t, _mm64(dpre.t(), x))
    check("shared db", db.t, dpre.sum(0), dpre.float().sum(0))


# ---- discriminator: dW1 [Kh, K] = dH^T x and dx (+)= -beta dH W1 ---------------------------------------------------
@pytest.mark.parametrize("engine", ["tf32", "tf32x3"])
@pytest.mark.parametrize("accumulate", [0, 1])
@pytest.mark.parametrize("rows,K", [(2560, 512), (1000, 256)])
def test_disc_bwd(rows, K, accumulate, engine):
    """ta3n_disc_bwd (Kh = K): at K = 256 the weight gradient is small and runs on the precise kernel under tf32x3."""
    L, lib = _lib()
    _engine(engine)
    g = torch.Generator().manual_seed(rows + K + accumulate)
    beta = 0.75
    x = grid((rows, K), 3, g)
    W1 = tf32_exact(torch.randn(K, K, generator=g) / math.sqrt(K))
    W2, gl = grid((2, K), 5, g), grid((rows, 2), 5, g)
    hidden = grid((rows, K), 3, g, relu=True)
    dx0 = grid((rows, K), 2, g) if accumulate else None
    dH = (_ref_dev(gl) @ _ref_dev(W2)) * (_ref_dev(hidden) > 0)
    _assert_tf32("disc dH / x / W1", dH, x, W1)
    d = _dev()
    t = {k: v.to(d) for k, v in dict(x=x, W1=W1, W2=W2, gl=gl, hidden=hidden).items()}
    dx, dW1, db1, dW2, db2 = _Out(rows, K), _Out(K, K), _Out(K), _Out(2, K), _Out(2)
    ws = _ws(lib.ta3n_disc_bwd_workspace_bytes(rows, K, K))
    dx0_d = None if dx0 is None else dx0.to(d)

    def run():
        for o in (dW1, db1, dW2, db2, dx):
            o.t.fill_(float("nan"))
        if accumulate:
            dx.t.copy_(dx0_d)
        L.check(lib.ta3n_disc_bwd(t["x"].data_ptr(), rows, K, K, t["W1"].data_ptr(), t["W2"].data_ptr(),
                                  t["hidden"].data_ptr(), t["gl"].data_ptr(), beta, dx.ptr(), accumulate, dW1.ptr(),
                                  db1.ptr(), dW2.ptr(), db2.ptr(), ws.data_ptr(), ws.numel(), _st()))

    L.timing_enable(True)
    try:
        names = _twice(run, [dx.t, dW1.t])
        sites = L.timing_report()
    finally:
        L.timing_enable(False)
    for o, w in ((dx, "dx"), (dW1, "dW1"), (db1, "db1"), (dW2, "dW2"), (db2, "db2")):
        o.check_guard(w)
    want = expect([G(K, K).seg(("dH",), ("x",), rows)], engine, False, False, arena=True)
    want += expect([G(rows, K).seg(("dH",), ("W1",), K)], engine, True, False)
    _assert_routes("disc_bwd", names, want, run)
    assert ("wgrad_small_x3" in sites) == _small_route(engine, K, K, rows), sorted(sites)
    ref_dx = -beta * _mm64(dH, W1) + (0 if dx0 is None else _ref_dev(dx0))
    tag = f"disc rows={rows} K={K} acc={accumulate} {engine}"
    tier_e(f"{tag} dW1 {dict(want)}", dW1.t, _mm64(dH.t(), x))
    tier_e(f"{tag} dx", dx.t, ref_dx)


# ---- TRN: dW per (scale, slot), dx per frame ------------------------------------------------------------------------
def _trn_setup(T, sampled):
    if sampled:
        tuples = _sampled_relations(T, seed=T)
        tab, keep = _ctable(T, tuples)
        return tuples, C.byref(tab), (tab, keep)
    from ta3n_b200.functional import relation_set
    rs = relation_set(T)
    return rs.tuples, rs.ref, rs


def _trn_plans(tuples, T, M, F, H, W_ptrs, x_ptr):
    """The weight-gradient plan (groups per (scale, slot)) and the data-gradient plan (groups per frame)."""
    wg, dg = [], []
    q0 = 0
    rel = []                                    # (q, scale i, tuple)
    for i, rels in enumerate(tuples):
        for tau in rels:
            rel.append((q0, i, tau))
            q0 += 1
    for i, rels in enumerate(tuples):
        s = len(rels[0])
        for j in range(s):
            gr = G(H, F)
            for q, ii, tau in rel:
                if ii == i:
                    gr.seg(("dz", q), ("x", x_ptr + 4 * tau[j] * F), M)
            wg.append(gr)
    for t in range(T):
        gr = G(M, F)
        for q, i, tau in rel:
            for j, f in enumerate(tau):
                if f == t:
                    gr.seg(("dz", q), ("W", W_ptrs[i] + 4 * j * F), H)
        if gr.segs:
            dg.append(gr)
    return wg, dg


def _trn_ref(tuples, x, W, G_, act_gate, relu_input, dx0):
    d = _dev()
    x64 = _ref_dev(x)
    xin = x64.clamp_min(0) if relu_input else x64
    M, T, F = x.shape
    dW = [torch.zeros(w.shape, dtype=torch.float64, device=d) for w in W]
    dx = torch.zeros(M, T, F, dtype=torch.float64, device=d)
    dzs, q = [], 0
    for i, rels in enumerate(tuples):
        Wi = _ref_dev(W[i])
        for tau in rels:
            dz = _ref_dev(G_[:, i, :]) * act_gate[q].to(d)
            dzs.append(dz)
            for j, f in enumerate(tau):
                dW[i][:, j * F:(j + 1) * F] += dz.t() @ xin[:, f, :]
                dx[:, f, :] += dz @ Wi[:, j * F:(j + 1) * F]
            q += 1
    if relu_input:
        dx = dx * (x64 > 0)
    if dx0 is not None:
        dx = dx + _ref_dev(dx0)
    return dW, dx, dzs


TRN = [(5, 48, 512, False), (9, 48, 512, False), (10, 48, 512, False), (13, 40, 512, False), (19, 48, 128, False),
       (20, 48, 128, False), (33, 72, 64, True)]


@pytest.mark.parametrize("engine", ["tf32", "tf32x3"])
@pytest.mark.parametrize("relu_input,accumulate_dx", [(0, 0), (1, 1), (0, 1), (1, 0)])
@pytest.mark.parametrize("T,M,F,sampled", TRN, ids=[f"T{c[0]}" for c in TRN])
def test_trn_bwd(T, M, F, sampled, relu_input, accumulate_dx, engine):
    """ta3n_trn_bwd: from T = 10 the weight gradient needs more than one launch (groups > 48, segments > 128); from
    T ~ 20 the data-gradient groups of some frames need more than 64 tensor maps and run on the SIMT engine.  With
    relu_input the weight gradient runs on the SIMT engine (ReLU on load) and the data gradient gates on x > 0."""
    L, lib = _lib()
    _engine(engine)
    H = 256
    tuples, tabref, _keep = _trn_setup(T, sampled)
    n_rel = sum(len(r) for r in tuples)
    g = torch.Generator().manual_seed(T * 1000 + relu_input * 10 + accumulate_dx)
    x = grid((M, T, F), 3, g)
    W = [tf32_exact(torch.randn(H, len(r[0]) * F, generator=g) / math.sqrt(len(r[0]) * F)) for r in tuples]
    act = grid((n_rel, M, H), 3, g, relu=True)
    Gr = grid((M, T - 1, H), 6, g)
    dx0 = grid((M, T, F), 2, g) if accumulate_dx else None
    d = _dev()
    xd, actd, Gd = x.to(d), act.to(d), Gr.to(d)
    Wd = [w.to(d) for w in W]
    dW = [_Out(*w.shape) for w in W]
    db = [_Out(H) for _ in W]
    dx = _Out(M, T, F)
    dx0_d = None if dx0 is None else dx0.to(d)
    ws = _ws(lib.ta3n_trn_bwd_workspace_bytes(M, F, H, tabref))
    W_pa, dW_pa, db_pa = _pa([w.data_ptr() for w in Wd]), _pa([o.ptr() for o in dW]), _pa([o.ptr() for o in db])

    def run():
        for o in dW + db:
            o.t.fill_(float("nan"))
        if accumulate_dx:
            dx.t.copy_(dx0_d)
        else:
            dx.t.fill_(float("nan"))
        L.check(lib.ta3n_trn_bwd(xd.data_ptr(), M, F, H, tabref, W_pa, relu_input, actd.data_ptr(), Gd.data_ptr(),
                                 dW_pa, db_pa, dx.ptr(), accumulate_dx, ws.data_ptr(), ws.numel(), _st()))

    names = _twice(run, [dx.t] + [o.t for o in dW])
    for o in dW + db + [dx]:
        o.check_guard("trn output")
    wg, dg = _trn_plans(tuples, T, M, F, H, [w.data_ptr() for w in Wd], xd.data_ptr())
    want = expect(wg, engine, False, False, relu_load=bool(relu_input), arena=True) + expect(dg, engine, True, False)
    _assert_routes(f"trn_bwd T={T}", names, want, run)
    if T >= 10 and not relu_input and not _small_route(engine, H, F, M):
        assert want["tc<false,false>"] >= 2, f"T={T}: the weight gradient should need several launches: {want}"
    if T >= 20:
        simt_frames = sum(len(gr.keys()) > MAX_MAPS for gr in dg)
        assert simt_frames > 0 and want["simt<true,false>"] >= 1, f"T={T}: no frame group beyond 64 maps"
    dW64, dx64, dzs = _trn_ref(tuples, x, W, Gr, [a > 0 for a in act], relu_input, dx0)
    _assert_tf32("trn dz / x / W", torch.stack(dzs), x, *W)
    tag = f"trn T={T} relu={relu_input} acc={accumulate_dx} {engine} {dict(want)}"
    slabs = lambda ws_: torch.cat([w.reshape(H, -1, F).transpose(0, 1) for w in ws_])  # noqa: E731
    tier_e(f"{tag} dW per (scale, slot)", slabs([o.t for o in dW]), slabs(dW64))
    tier_e(f"{tag} dx per frame", dx.t.transpose(0, 1), dx64.transpose(0, 1))
    first = [sum(len(r) for r in tuples[:i]) for i in range(len(tuples) + 1)]
    db64 = torch.stack([sum(dzs[q].sum(0) for q in range(first[i], first[i + 1])) for i in range(len(tuples))])
    assert torch.equal(torch.stack([o.t for o in db]).double(), db64), "db: sums of grid values must be exact"


# ---- relation discriminators: dW1_i = dHid_i^T feat_rel_i, d_feat_rel_i = (a_i + 1) G - beta dHid_i W1_i ----------
def _relattn_exact(M, R, H, use_attn, g):
    fr = grid((M, R, H), 3, g)
    W1 = [tf32_exact(torch.randn(H, H, generator=g) / math.sqrt(H)) for _ in range(R)]
    W2 = [grid((2, H), 5, g) for _ in range(R)]
    hidden = grid((R, M, H), 3, g, relu=True)
    gp = grid((M, R, 2), 5, g)
    Gv = grid((M, H), 4, g)
    attn = grid((M, R), 5, g).abs() if use_attn == 2 else fr[:, :, 0].clone()
    return fr, W1, W2, hidden, gp, Gv, attn


def _relattn_call(lib, t, M, R, H, use_attn, beta, dfr, dW1, db1, dW2, db2, ws, g_attn=None):
    pa = lambda ts: _pa([v.data_ptr() for v in ts])     # noqa: E731
    return lib.ta3n_relattn_bwd(t["fr"].data_ptr(), M, R, H, pa(t["W1"]), pa(t["W2"]), use_attn, t["hidden"].data_ptr(),
                                t["pred"].data_ptr(), t["attn"].data_ptr(), t["G"].data_ptr(), t["gp"].data_ptr(),
                                None if g_attn is None else g_attn.data_ptr(), beta, dfr.ptr(),
                                _pa([o.ptr() for o in dW1]), _pa([o.ptr() for o in db1]),
                                _pa([o.ptr() for o in dW2]), _pa([o.ptr() for o in db2]), ws.data_ptr(), ws.numel(),
                                _st())


def _relattn_plans(M, R, H, fr_ptr, W1_ptrs):
    wg = [G(H, H).seg(("dHid", i), ("fr", fr_ptr + 4 * i * H), M) for i in range(R)]
    dg = [G(M, H).seg(("dHid", i), ("W1", W1_ptrs[i]), H) for i in range(R)]
    return wg, dg


@pytest.mark.parametrize("engine", ["tf32", "tf32x3"])
@pytest.mark.parametrize("use_attn", [0, 2])
@pytest.mark.parametrize("R", [1, 2, 5, 8, 9])
def test_relattn_bwd(R, use_attn, engine):
    """ta3n_relattn_bwd: the weight gradient reads feat_rel[:, i, :] (ld = R H); with use_attn = 2 the data gradient's
    epilogue adds (a + 1) G."""
    L, lib = _lib()
    _engine(engine)
    M, H, beta = 300, 256, 0.75
    g = torch.Generator().manual_seed(R * 10 + use_attn)
    fr, W1, W2, hidden, gp, Gv, attn = _relattn_exact(M, R, H, use_attn, g)
    gate = _ref_dev(hidden) > 0
    dHid = torch.stack([(_ref_dev(gp[:, i, 0:1]) * _ref_dev(W2[i][0]) + _ref_dev(gp[:, i, 1:2]) * _ref_dev(W2[i][1]))
                        for i in range(R)]) * gate
    _assert_tf32("relattn dHid / feat_rel / W1", dHid, fr, *W1)
    d = _dev()
    t = dict(fr=fr.to(d), W1=[w.to(d) for w in W1], W2=[w.to(d) for w in W2], hidden=hidden.to(d),
             pred=torch.zeros(M, R, 2, device=d), attn=attn.to(d), G=Gv.to(d), gp=gp.to(d))
    dfr = _Out(M, R, H)
    dW1, db1 = [_Out(H, H) for _ in range(R)], [_Out(H) for _ in range(R)]
    dW2, db2 = [_Out(2, H) for _ in range(R)], [_Out(2) for _ in range(R)]
    ws = _ws(lib.ta3n_relattn_bwd_workspace_bytes(M, R, H))

    def run():
        for o in [dfr] + dW1 + db1 + dW2 + db2:
            o.t.fill_(float("nan"))
        L.check(_relattn_call(lib, t, M, R, H, use_attn, beta, dfr, dW1, db1, dW2, db2, ws))

    names = _twice(run, [dfr.t] + [o.t for o in dW1])
    for o in [dfr] + dW1 + db1 + dW2 + db2:
        o.check_guard("relattn output")
    wg, dg = _relattn_plans(M, R, H, t["fr"].data_ptr(), [w.data_ptr() for w in t["W1"]])
    want = expect(wg, engine, False, False, arena=True) + expect(dg, engine, True, False)
    _assert_routes("relattn_bwd", names, want, run)
    rowscale = (_ref_dev(attn) + 1) if use_attn == 2 else torch.ones(M, R, dtype=torch.float64, device=d)
    ref_dfr = torch.stack([rowscale[:, i:i + 1] * _ref_dev(Gv) - beta * _mm64(dHid[i], W1[i]) for i in range(R)])
    ref_dW1 = torch.stack([_mm64(dHid[i].t(), fr[:, i, :]) for i in range(R)])
    tag = f"relattn R={R} use_attn={use_attn} {engine} {dict(want)}"
    tier_e(f"{tag} dW1 per relation", torch.stack([o.t for o in dW1]), ref_dW1)
    tier_e(f"{tag} d_feat_rel per relation", dfr.t.transpose(0, 1), ref_dfr)


# ---- video head: dWc [C, H] = g_pred^T dropped ----------------------------------------------------------------------
@pytest.mark.parametrize("engine", ["tf32", "tf32x3"])
@pytest.mark.parametrize("Cn", [64, 100, 33])
def test_video_head_bwd(Cn, engine):
    """ta3n_video_head_bwd with a dropout keep mask: C = 64 and 100 take the GEMM route, C = 33 (ld of g_pred not a
    multiple of 4) the SIMT engine."""
    from ta3n_b200.functional import DropSpec
    L, lib = _lib()
    _engine(engine)
    M, H, p, scale = 256, 256, 0.5, -0.5
    g = torch.Generator().manual_seed(Cn)
    dropped, Wc, gp = grid((M, H), 3, g), grid((Cn, H), 5, g), grid((M, Cn), 5, g)
    keep = (torch.rand(M, H, generator=g) < 0.5).to(torch.uint8)
    _assert_tf32("video head g_pred / dropped", gp, dropped)
    d = _dev()
    dd, Wd, gpd, keepd = dropped.to(d), Wc.to(d), gp.to(d), keep.to(d)
    dc = DropSpec(p, keepd).cstruct()
    dfv, dWc, dbc = _Out(M, H), _Out(Cn, H), _Out(Cn)
    ws = _ws(lib.ta3n_video_head_bwd_workspace_bytes(M, H, Cn))

    def run():
        for o in (dfv, dWc, dbc):
            o.t.fill_(float("nan"))
        L.check(lib.ta3n_video_head_bwd(dd.data_ptr(), M, H, Cn, Wd.data_ptr(), C.byref(dc), gpd.data_ptr(), None, None,
                                        scale, dfv.ptr(), dWc.ptr(), dbc.ptr(), ws.data_ptr(), ws.numel(), _st()))

    names = _twice(run, [dfv.t, dWc.t, dbc.t])
    for o, w in ((dfv, "d_feat_video"), (dWc, "dWc"), (dbc, "dbc")):
        o.check_guard(w)
    gr = G(Cn, H).seg(("gp", gpd.data_ptr()), ("dropped", dd.data_ptr()), M, ok=_aligned(gpd.data_ptr(), Cn))
    want = expect([gr], engine, False, False, arena=True)
    _assert_routes("video_head_bwd", names, want, run)
    ref_dfv = (_ref_dev(gp) @ _ref_dev(Wc)) * scale * _ref_dev(keep) / (1 - p)
    tier_e(f"video head C={Cn} {engine} dWc {dict(want)}", dWc.t, _mm64(gp.t(), dropped))
    tier_e(f"video head C={Cn} {engine} d_feat_video", dfv.t, ref_dfv)


# ---- all of them deferred into one wgrad_all plan -------------------------------------------------------------------
@pytest.mark.parametrize("engine", ["tf32", "tf32x3"])
@pytest.mark.parametrize("T", [5, 10])
def test_deferred_weight_gradients(T, engine):
    """The backward entry points between ta3n_wgrad_defer_begin and _flush at cfg2-like sizes (256 + 256 videos, D =
    2048, F = 512, H = 256; C = 64 so that the video head has a GEMM): their weight gradients run as one mixed
    M-major x N-major plan, the small ones on the precise kernel under tf32x3."""
    from ta3n_b200.functional import DropSpec, relation_set
    L, lib = _lib()
    _engine(engine)
    Mv, D, F, H, Cn, beta = 512, 2048, 512, 256, 64, 0.75
    rows = Mv * T
    R = T - 1
    g = torch.Generator().manual_seed(T)
    d = _dev()
    want = Counter()
    wgrad_groups = []
    checks = []
    keepalive = []

    # shared layer
    x, feat, dfeat, gext, dpre = _shared_inputs(rows // 2, rows // 2, D, F, 0.5, True, g)
    _assert_tf32("deferred shared", dpre, x)
    xs, xt = x[:rows // 2].contiguous().to(d), x[rows // 2:].contiguous().to(d)
    feat_d, dfeat_d, gext_d = feat.to(d), dfeat.to(d), gext.to(d)
    dfb = torch.empty_like(dfeat_d)
    sh_dW, sh_db = _Out(F, D), _Out(F)
    sh_ws = _ws(lib.ta3n_shared_fc_bwd_workspace_bytes(rows, D, F))
    wgrad_groups.append(_shared_plan(F, D, rows // 2, rows // 2, xs, xt))
    checks.append(("shared dW", sh_dW, lambda: _mm64(dpre.t(), x)))

    # frame discriminator (rows x F, Kh = F) and video discriminator (Mv x H, Kh = H)
    discs = []
    for name, drows, K in (("frame disc", rows, F), ("video disc", Mv, H)):
        dx_ = grid((drows, K), 3, g)
        W1 = tf32_exact(torch.randn(K, K, generator=g) / math.sqrt(K))
        W2, gl = grid((2, K), 5, g), grid((drows, 2), 5, g)
        hid = grid((drows, K), 3, g, relu=True)
        dH = (_ref_dev(gl) @ _ref_dev(W2)) * (_ref_dev(hid) > 0)
        _assert_tf32(name, dH, dx_, W1)
        t = [v.to(d) for v in (dx_, W1, W2, hid, gl)]
        outs = [_Out(drows, K), _Out(K, K), _Out(K), _Out(2, K), _Out(2)]
        ws_ = _ws(lib.ta3n_disc_bwd_workspace_bytes(drows, K, K))
        discs.append((drows, K, t, outs, ws_))
        wgrad_groups.append(G(K, K).seg((name, "dH"), (name, "x"), drows))
        want += expect([G(drows, K).seg((name, "dH"), (name, "W1"), K)], engine, True, False)
        checks.append((f"{name} dW1", outs[1], lambda dH=dH, dx_=dx_: _mm64(dH.t(), dx_)))
        checks.append((f"{name} dx", outs[0], lambda dH=dH, W1=W1: -beta * _mm64(dH, W1)))

    # TRN
    rs = relation_set(T)
    tx = grid((Mv, T, F), 3, g)
    tW = [tf32_exact(torch.randn(H, len(r[0]) * F, generator=g) / math.sqrt(len(r[0]) * F)) for r in rs.tuples]
    tact = grid((rs.n_rel, Mv, H), 3, g, relu=True)
    tG = grid((Mv, R, H), 6, g)
    txd, tWd, tactd, tGd = tx.to(d), [w.to(d) for w in tW], tact.to(d), tG.to(d)
    t_dW, t_db, t_dx = [_Out(*w.shape) for w in tW], [_Out(H) for _ in tW], _Out(Mv, T, F)
    t_ws = _ws(lib.ta3n_trn_bwd_workspace_bytes(Mv, F, H, rs.ref))
    wg, dg = _trn_plans(rs.tuples, T, Mv, F, H, [w.data_ptr() for w in tWd], txd.data_ptr())
    wgrad_groups += wg
    want += expect(dg, engine, True, False)
    tdW64, tdx64, tdzs = _trn_ref(rs.tuples, tx, tW, tG, [a > 0 for a in tact], 0, None)
    _assert_tf32("deferred trn", torch.stack(tdzs), tx, *tW)

    # relation discriminators (use_attn = 2) and the video head
    fr, rW1, rW2, rhid, rgp, rG, rattn = _relattn_exact(Mv, R, H, 2, g)
    rt = dict(fr=fr.to(d), W1=[w.to(d) for w in rW1], W2=[w.to(d) for w in rW2], hidden=rhid.to(d),
              pred=torch.zeros(Mv, R, 2, device=d), attn=rattn.to(d), G=rG.to(d), gp=rgp.to(d))
    r_dfr = _Out(Mv, R, H)
    r_dW1, r_db1 = [_Out(H, H) for _ in range(R)], [_Out(H) for _ in range(R)]
    r_dW2, r_db2 = [_Out(2, H) for _ in range(R)], [_Out(2) for _ in range(R)]
    r_ws = _ws(lib.ta3n_relattn_bwd_workspace_bytes(Mv, R, H))
    rwg, rdg = _relattn_plans(Mv, R, H, rt["fr"].data_ptr(), [w.data_ptr() for w in rt["W1"]])
    wgrad_groups += rwg
    want += expect(rdg, engine, True, False)
    rdHid = torch.stack([(_ref_dev(rgp[:, i, 0:1]) * _ref_dev(rW2[i][0]) + _ref_dev(rgp[:, i, 1:2]) *
                          _ref_dev(rW2[i][1])) for i in range(R)]) * (_ref_dev(rhid) > 0)
    _assert_tf32("deferred relattn", rdHid, fr, *rW1)

    vdrop, vW, vgp = grid((Mv, H), 3, g), grid((Cn, H), 5, g), grid((Mv, Cn), 5, g)
    vkeep = (torch.rand(Mv, H, generator=g) < 0.5).to(torch.uint8).to(d)
    vdc = DropSpec(0.5, vkeep).cstruct()
    vd, vWd, vgpd = vdrop.to(d), vW.to(d), vgp.to(d)
    v_dfv, v_dWc, v_dbc = _Out(Mv, H), _Out(Cn, H), _Out(Cn)
    v_ws = _ws(lib.ta3n_video_head_bwd_workspace_bytes(Mv, H, Cn))
    wgrad_groups.append(G(Cn, H).seg(("vh", "gp"), ("vh", "dropped"), Mv))
    want += expect(wgrad_groups, engine, False, False, arena=True)
    keepalive += [vdc, vkeep]

    fws = _ws(lib.ta3n_wgrad_defer_workspace_bytes())
    outs = ([sh_dW, sh_db] + [o for *_, outs_, _w in discs for o in outs_] + t_dW + t_db + [t_dx, r_dfr] + r_dW1 +
            r_db1 + r_dW2 + r_db2 + [v_dfv, v_dWc, v_dbc])

    def run():
        for o in outs:
            o.t.fill_(float("nan"))
        dfb.copy_(dfeat_d)
        L.check(lib.ta3n_wgrad_defer_begin())
        L.check(_shared_call(lib, xs, rows // 2, xt, rows // 2, D, F, feat_d, dfb, gext_d, 0.5, sh_dW, sh_db, sh_ws))
        for drows, K, t, o, ws_ in discs:
            L.check(lib.ta3n_disc_bwd(t[0].data_ptr(), drows, K, K, t[1].data_ptr(), t[2].data_ptr(),
                                      t[3].data_ptr(), t[4].data_ptr(), beta, o[0].ptr(), 0, o[1].ptr(), o[2].ptr(),
                                      o[3].ptr(), o[4].ptr(), ws_.data_ptr(), ws_.numel(), _st()))
        L.check(lib.ta3n_trn_bwd(txd.data_ptr(), Mv, F, H, rs.ref, _pa([w.data_ptr() for w in tWd]), 0,
                                 tactd.data_ptr(), tGd.data_ptr(), _pa([o.ptr() for o in t_dW]),
                                 _pa([o.ptr() for o in t_db]), t_dx.ptr(), 0, t_ws.data_ptr(), t_ws.numel(), _st()))
        L.check(_relattn_call(lib, rt, Mv, R, H, 2, beta, r_dfr, r_dW1, r_db1, r_dW2, r_db2, r_ws))
        L.check(lib.ta3n_video_head_bwd(vd.data_ptr(), Mv, H, Cn, vWd.data_ptr(), C.byref(vdc), vgpd.data_ptr(), None,
                                        None, 1.0, v_dfv.ptr(), v_dWc.ptr(), v_dbc.ptr(), v_ws.data_ptr(),
                                        v_ws.numel(), _st()))
        L.check(lib.ta3n_wgrad_defer_flush(fws.data_ptr(), fws.numel(), _st()))

    names = _twice(run, [o.t for o in outs])
    for o in outs:
        o.check_guard("deferred output")
    _assert_routes(f"deferred T={T}", names, want, run)
    tag = f"deferred T={T} {engine}"
    for what, o, ref in checks:
        tier_e(f"{tag} {what}", o.t, ref())
    slabs = lambda ws_: torch.cat([w.reshape(H, -1, F).transpose(0, 1) for w in ws_])  # noqa: E731
    tier_e(f"{tag} trn dW per (scale, slot)", slabs([o.t for o in t_dW]), slabs(tdW64))
    tier_e(f"{tag} trn dx per frame", t_dx.t.transpose(0, 1), tdx64.transpose(0, 1))
    tier_e(f"{tag} relattn dW1 per relation", torch.stack([o.t for o in r_dW1]),
           torch.stack([_mm64(rdHid[i].t(), fr[:, i, :]) for i in range(R)]))
    ref_dfr = torch.stack([(_ref_dev(rattn[:, i:i + 1]) + 1) * _ref_dev(rG) - beta * _mm64(rdHid[i], rW1[i])
                           for i in range(R)])
    tier_e(f"{tag} relattn d_feat_rel per relation", r_dfr.t.transpose(0, 1), ref_dfr)
    tier_e(f"{tag} video head dWc", v_dWc.t, _mm64(vgp.t(), vdrop))


# ------------------------------------------------------------------------------------------------
# B'. tier R where the operands come from tanh, softmax or entropy arithmetic
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("engine", ["tf32", "tf32x3"])
def test_relattn_bwd_transattn_raw(engine):
    """ta3n_relattn_bwd with use_attn = 1 (dHid from the entropy attention's gradient), forward on the exact engine."""
    from tests.test_rowops_fp32 import _relattn_inputs, _relattn_ref
    L, lib = _lib()
    M, R, H, beta = 300, 8, 256, 0.6
    fr, W1, b1, W2, b2, Gv, gp, ga, _ = _relattn_inputs(M, R, H, seed=3)
    d = _dev()
    dev = lambda ts: [v.to(d) for v in ts]              # noqa: E731
    W1d, b1d, W2d, b2d = dev(W1), dev(b1), dev(W2), dev(b2)
    pa = lambda ts: _pa([v.data_ptr() for v in ts])     # noqa: E731
    frd = fr.to(d)
    hid, pred, attn, fv = Buf(R, M, H), Buf(M, R, 2), Buf(M, R), Buf(M, H)
    _engine("fp32")
    L.check(lib.ta3n_relattn_fwd(frd.data_ptr(), M, R, H, pa(W1d), pa(b1d), pa(W2d), pa(b2d), 1, hid.p, pred.p,
                                 attn.p, fv.p, _st()))
    _engine(engine)
    t = dict(fr=frd, W1=W1d, W2=W2d, hidden=hid.t, pred=pred.t, attn=attn.t, G=Gv.to(d), gp=gp.to(d))
    dfr = _Out(M, R, H)
    dW1, db1 = [_Out(H, H) for _ in range(R)], [_Out(H) for _ in range(R)]
    dW2, db2 = [_Out(2, H) for _ in range(R)], [_Out(2) for _ in range(R)]
    ws = _ws(lib.ta3n_relattn_bwd_workspace_bytes(M, R, H))
    gad = ga.to(d)

    def run():
        for o in [dfr] + dW1 + db1 + dW2 + db2:
            o.t.fill_(float("nan"))
        L.check(_relattn_call(lib, t, M, R, H, 1, beta, dfr, dW1, db1, dW2, db2, ws, g_attn=gad))

    names = _twice(run, [dfr.t] + [o.t for o in dW1])
    for o in [dfr] + dW1:
        o.check_guard("relattn output")
    wg, dg = _relattn_plans(M, R, H, frd.data_ptr(), [w.data_ptr() for w in W1d])
    want = expect(wg, engine, False, False, arena=True) + expect(dg, engine, True, False)
    _assert_routes("relattn_bwd use_attn=1", names, want, run)
    r64 = _relattn_ref(torch.float64, fr, W1, b1, W2, b2, [h > 0 for h in hid.cpu()], 1, beta, None, Gv, gp, ga)
    got_dW1 = torch.stack([o.t for o in dW1])
    if _small_route(engine, H, H, M):
        tier_e(f"relattn use_attn=1 {engine} dW1 (precise)", got_dW1, r64["dW1"])
    else:
        tier_r(f"relattn use_attn=1 {engine} dW1", got_dW1, r64["dW1"])
    tier_r(f"relattn use_attn=1 {engine} d_feat_rel", dfr.t.transpose(0, 1), r64["d_feat_rel"].transpose(0, 1))


@pytest.mark.parametrize("engine", ["tf32", "tf32x3"])
@pytest.mark.parametrize("M,R", [(256, 8), (400, 9)])
def test_general_attn_bwd_raw(M, R, engine):
    """ta3n_general_attn_bwd (d_pre from tanh and the softmax over relations), forward on the exact engine; dW1 has K
    = M R: 2048 (small, precise under tf32x3) and 3600 (plain)."""
    from tests.test_rowops_fp32 import _general_ref
    L, lib = _lib()
    H = 256
    g = torch.Generator().manual_seed(M + R)
    # feat_rel of mixed sign: the softmax gradient sums to 0 over the relations, so with a positive feat_rel dW1
    # would be a cancelling sum whose relative error is no longer that of one tf32 product
    fr = torch.randn(M, R, H, generator=g)
    W1, b1 = torch.randn(H, H, generator=g) / math.sqrt(H), 0.1 * torch.randn(H, generator=g)
    w2, b2 = 3 * torch.randn(1, H, generator=g) / math.sqrt(H), torch.randn(1, generator=g)
    S0, D0, Gv = torch.zeros(M, H), torch.zeros(M, R, H), torch.randn(M, H, generator=g)
    d = _dev()
    frd, W1d, b1d, w2d, b2d = (v.to(d) for v in (fr, W1, b1, w2, b2))
    hid, attn, fv = Buf(M * R, H), Buf(M, R), Buf(M, H, init=S0.to(d))
    _engine("fp32")
    L.check(lib.ta3n_general_attn_fwd(frd.data_ptr(), M, R, H, W1d.data_ptr(), b1d.data_ptr(), w2d.data_ptr(),
                                      b2d.data_ptr(), hid.p, attn.p, fv.p, _st()))
    _engine(engine)
    dfr = _Out(M, R, H)
    dW1, db1, dw2, db2 = _Out(H, H), _Out(H), _Out(1, H), _Out(1)
    Gd = Gv.to(d)
    ws = _ws(lib.ta3n_general_attn_bwd_workspace_bytes(M, R, H))

    def run():
        dfr.t.zero_()                                   # EPI_ACCUM: d_feat_rel += d_pre W1 onto known zeros
        for o in (dW1, db1, dw2, db2):
            o.t.fill_(float("nan"))
        L.check(lib.ta3n_general_attn_bwd(frd.data_ptr(), M, R, H, W1d.data_ptr(), w2d.data_ptr(), hid.p, attn.p,
                                          Gd.data_ptr(), None, dfr.ptr(), dW1.ptr(), db1.ptr(), dw2.ptr(), db2.ptr(),
                                          ws.data_ptr(), ws.numel(), _st()))

    names = _twice(run, [dfr.t, dW1.t])
    for o, w in ((dfr, "d_feat_rel"), (dW1, "dW1"), (db1, "db1"), (dw2, "dw2"), (db2, "db2")):
        o.check_guard(w)
    want = expect([G(H, H).seg(("d_pre",), ("fr",), M * R)], engine, False, False, arena=True)
    want += expect([G(M * R, H).seg(("d_pre",), ("W1",), H)], engine, True, False)
    _assert_routes("general_attn_bwd", names, want, run)
    r64 = _general_ref(torch.float64, fr, W1, b1, w2, b2, S0, D0, Gv, None)
    if _small_route(engine, H, H, M * R):
        tier_e(f"general attn M={M} R={R} {engine} dW1 (precise)", dW1.t, r64["dW1"])
    else:
        tier_r(f"general attn M={M} R={R} {engine} dW1", dW1.t, r64["dW1"])
    tier_r(f"general attn M={M} R={R} {engine} d_feat_rel", dfr.t.view(M * R, H), r64["d_feat_rel"].view(M * R, H))
