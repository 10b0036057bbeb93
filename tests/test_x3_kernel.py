"""The precise tensor-core kernel (tf32x3) in the operand layouts other than the forward K-major x K-major one, which
the full-size training-step tests cover: fp32-grade results against fp64, with K long enough for several 8-slab
accumulation chunks, an odd slab count and ragged tile edges.

  M-major x N-major (weight gradients of the 256 x 256 discriminator layers): through ta3n_gemm_ex, whose small
                     M-major x N-major products run on the precise kernel under tf32x3.
  K-major x N-major (data gradients with TA3N_X3_DGRAD=1): through ta3n_disc_bwd in a child process, because the
                     library reads that variable once.

A plain tf32 product is ~3e-4 off normwise; the bound below is 15x tighter.
"""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
X3_TOL = 2e-5


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).norm() / b.norm()).item()


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
