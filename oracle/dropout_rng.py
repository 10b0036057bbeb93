"""Host restatement of the counter-based dropout RNG  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

The kernels never store a dropout mask: every keep decision is recomputed from (seed, step, element) by
``rng_keep`` of ``ta3n_b200/csrc/common.cuh``.  This module restates that function in numpy ``uint64`` (wrapping
arithmetic, bit for bit) and rebuilds the keep masks a forward drew, in the ``masks`` format of
``ta3n_oracle.forward`` / ``train_step`` ('i_source' (Bs*T,F), 'i_target', 'v_source' (Bs,H), 'v_target'), so that
a dropout-on step of the CUDA path can be compared with the fp64 network evaluated on the same masks.

Conventions of the library (what the helpers below encode):
  * shared layer: element e = row-major index into the [(Bs+Bt)*T, F] feature tensor, source rows first; target
    rows start at Bs*T*F, Bs being the batch size the step was built for (also when a shorter batch is loaded);
  * video dropout: e = m*H + h over [(Bs+Bt), H] (H = F under avgpool);
  * TrainStep seeds: drop_i uses seed ^ (rank * 0x9E3779B97F4A7C15) masked to 63 bits, drop_v that value ^ 0x9E3779B9;
    the step value is the device counter as the kernels read it (``TrainStep`` mode 'legacy' increments it before
    the forward, 'phased' after the backward);
  * ``VideoModel.forward``: one ``model._rng.getrandbits(63)`` for dropout_i, then one for dropout_v, each only for a
    rate > 0; step 0 (no device counter).
"""
from __future__ import annotations

import random
from typing import Dict, Optional, Tuple

import numpy as np
import torch

_U64 = np.uint64
_GOLDEN = 0x9E3779B97F4A7C15
_IDX_MUL = 0xD6E8FEB86659FD93
_SEED_MASK = (1 << 63) - 1


def _u64(x) -> np.ndarray:
    return np.asarray(x, dtype=np.uint64)


def mix64(z) -> np.ndarray:
    """splitmix64 finaliser (common.cuh mix64), elementwise on uint64."""
    z = _u64(z)
    with np.errstate(over="ignore"):
        z = (z ^ (z >> _U64(30))) * _U64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> _U64(27))) * _U64(0x94D049BB133111EB)
    return z ^ (z >> _U64(31))


def rng_hash4(seed: int, step: int, idx4) -> np.ndarray:
    """One 64-bit hash per group of four consecutive elements (common.cuh rng_hash4)."""
    seed, step = int(seed) & (2 ** 64 - 1), int(step) & (2 ** 64 - 1)
    key = (seed + _GOLDEN * (step + 1)) & (2 ** 64 - 1)          # same wrap-around as the device's uint64 arithmetic
    with np.errstate(over="ignore"):
        return mix64(mix64(_u64(key)) ^ (_u64(idx4) * _U64(_IDX_MUL)))


def threshold(p: float) -> int:
    """(uint32)(p * 65536 + 0.5) in float32, as the device computes it from the float32 rate it is given."""
    v = np.float32(p) * np.float32(65536.0) + np.float32(0.5)
    return int(np.uint32(v))


def keep(seed: int, step: int, e, p: float) -> np.ndarray:
    """Keep decision (bool) of element(s) e: 16 bits of the quad's hash >= threshold(p)."""
    e = _u64(e)
    h = rng_hash4(seed, step, e >> _U64(2))
    bits = (h >> (_U64(16) * (e & _U64(3)))) & _U64(0xFFFF)
    return bits >= _U64(threshold(p))


def _mask(seed: int, step: int, start: int, rows: int, cols: int, p: float) -> torch.Tensor:
    e = np.arange(rows * cols, dtype=np.uint64) + _U64(start)
    return torch.from_numpy(keep(seed, step, e, p).astype(np.uint8).reshape(rows, cols))


def shared_masks(seed: int, step: int, Bs: int, Bt: int, T: int, F: int, p: float,
                 ns: Optional[int] = None, nt: Optional[int] = None) -> Dict[str, torch.Tensor]:
    """Keep masks of the shared layer's dropout for the first ns source / nt target videos (default: all) of a
    launch over Bs + Bt videos."""
    ns = Bs if ns is None else ns
    nt = Bt if nt is None else nt
    return {"i_source": _mask(seed, step, 0, ns * T, F, p),
            "i_target": _mask(seed, step, Bs * T * F, nt * T, F, p)}


def video_masks(seed: int, step: int, Bs: int, Bt: int, H: int, p: float,
                ns: Optional[int] = None, nt: Optional[int] = None) -> Dict[str, torch.Tensor]:
    """Keep masks of dropout_v (e = m*H + h, source videos first)."""
    ns = Bs if ns is None else ns
    nt = Bt if nt is None else nt
    return {"v_source": _mask(seed, step, 0, ns, H, p), "v_target": _mask(seed, step, Bs * H, nt, H, p)}


def train_step_seeds(seed: int = 0x5EED, rank: int = 0) -> Tuple[int, int]:
    """(drop_i seed, drop_v seed) of ``TrainStep(seed=seed)`` on data-parallel rank ``rank``."""
    s = (int(seed) ^ (int(rank) * _GOLDEN)) & _SEED_MASK
    return s, s ^ 0x9E3779B9


def path_masks(seed_i: Optional[int], seed_v: Optional[int], step: int, Bs: int, Bt: int, T: int, F: int, H: int,
               p_i: float, p_v: float, ns: Optional[int] = None, nt: Optional[int] = None) -> Dict[str, torch.Tensor]:
    """The oracle's ``masks`` for one forward of the path (a rate of 0 contributes no key)."""
    out: Dict[str, torch.Tensor] = {}
    if p_i > 0:
        out.update(shared_masks(seed_i, step, Bs, Bt, T, F, p_i, ns, nt))
    if p_v > 0:
        out.update(video_masks(seed_v, step, Bs, Bt, H, p_v, ns, nt))
    return out


def train_step_masks(step: int, Bs: int, Bt: int, T: int, F: int, H: int, p_i: float, p_v: float,
                     seed: int = 0x5EED, rank: int = 0, ns: Optional[int] = None,
                     nt: Optional[int] = None) -> Dict[str, torch.Tensor]:
    """Masks of one ``TrainStep`` replay whose kernels read the step counter as ``step``."""
    si, sv = train_step_seeds(seed, rank)
    return path_masks(si, sv, step, Bs, Bt, T, F, H, p_i, p_v, ns, nt)


def model_forward_seeds(rng_state, p_i: float, p_v: float) -> Tuple[Optional[int], Optional[int]]:
    """Seeds one ``VideoModel.forward`` draws from ``model._rng`` whose state before the call was ``rng_state``."""
    r = random.Random()
    r.setstate(rng_state)
    si = r.getrandbits(63) if p_i > 0 else None
    sv = r.getrandbits(63) if p_v > 0 else None
    return si, sv
