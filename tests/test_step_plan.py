"""Host-side checks of the step program (no GPU): ta3n_step_workspace_bytes builds the program for a descriptor with
placeholder pointers and sizes its workspace without a CUDA call."""
import ctypes as C

import pytest

from ta3n_b200 import _lib
from ta3n_b200 import functional as TF


def _desc(Bs, Bt, T, C_, F=512, H=256, D=2048, drop=0.5):
    d = _lib.StepDesc()
    d.Bs, d.Bt, d.T, d.D, d.F, d.H, d.C = Bs, Bt, T, D, F, H, C_
    d.use_attn, d.loss_flags, d.gamma = 1, 15, 0.003
    d.domain_weight[0], d.domain_weight[1] = 1.0, 1.0
    rs = TF.relation_set(T)
    d.tab = C.pointer(rs.ctable)
    keep = [rs]
    fake = 1 << 30                      # never dereferenced by the host-only planner; 256-byte aligned

    def nxt():
        nonlocal fake
        fake += 1 << 26
        return fake

    R = T - 1
    for name, ctype in d._fields_:
        if ctype is C.c_void_p and name not in ("class_weight", "valid_rows"):
            setattr(d, name, nxt())
        elif ctype == C.POINTER(C.c_void_p):
            arr = (C.c_void_p * R)(*[nxt() for _ in range(R)])
            keep.append(arr)
            setattr(d, name, arr)
    d.drop_i.p = drop
    d.drop_i.seed = 1
    d.drop_i.keep = None
    d.drop_i.step_dev = nxt()
    d.drop_v.p = drop
    d.drop_v.seed = 2
    d.drop_v.keep = None
    d.drop_v.step_dev = nxt()
    d.workspace_bytes = 1 << 40
    return d, keep


def _fixed_scratch_bytes(Bs, Bt, T, C_, F=512, H=256):
    """The scratch tensors the step program carves first (csrc/step_plan.cuh), each rounded to 64 floats."""
    M, R, n_rel = Bs + Bt, T - 1, TF.relation_set(T).n_rel
    r = lambda n: -(-n // 64) * 64
    return 4 * (r(M * C_) + r(M * 2) + r(M * T * 2) + 2 * r(M * R * 2) + 3 * r(M * H) + r(R * M * H) +
                2 * r(M * T * F) + r(M * R * H) + r(n_rel * M * H) + r(M) + r(M * T))


@pytest.mark.parametrize("Bs,Bt,T,C_", [(256, 256, 5, 12), (512, 512, 5, 30), (128, 128, 9, 12), (8, 8, 5, 5),
                                        (3, 1, 5, 7), (60, 51, 3, 11), (130, 127, 5, 12)])
def test_workspace_covers_scratch_and_column_sums(Bs, Bt, T, C_):
    lib = _lib.load()
    d, keep = _desc(Bs, Bt, T, C_)
    n = lib.ta3n_step_workspace_bytes(C.byref(d))
    assert n > 0, lib.ta3n_last_error()
    # the column sums' partials follow the fixed scratch
    assert n > _fixed_scratch_bytes(Bs, Bt, T, C_)


def test_invalid_descriptor_is_rejected():
    lib = _lib.load()
    d, keep = _desc(8, 8, 5, 5, H=100)
    assert lib.ta3n_step_workspace_bytes(C.byref(d)) == 0
    assert b"H in {128, 256}" in lib.ta3n_last_error()
