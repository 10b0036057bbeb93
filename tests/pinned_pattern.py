"""Shared helpers of the step tests that pin the ReLU pattern a TrainStep realised.

A handful of the ReLU units of a step have pre-activations within rounding of zero, and every implementation decides
some of them differently from the fp64 network; at the full size ONE such unit moves the shared layer's weight
gradient by ~1e-3 normwise (test_gpu_parity.py).  These helpers read the pattern the kernels realised out of the step's
buffer pool, in the oracle's ``gates`` format, count the units where it differs from the fp64 pattern, and compare
every gradient against the fp64 oracle evaluated on that pattern.
"""
import torch

from tests.golden_util import abs_err, assert_close

# The rounding floor of the domain heads' bias gradients (golden_util uses it for the same sums): their source and
# target halves, O(0.25) each at the full size, cancel to ~1e-7, so any fp32 summation order is off by ~1e-8, and the
# fp32 restatement's own error -- one sample of that rounding -- can come out luckily small.
BIAS_SUM_FLOOR = 4e-9


def real_rows(Bs, ns, nt, T):
    """(frames, videos): the real rows of a pool tensor of the captured batch Bs + Bt (target rows start at Bs), on
    the host -- frame-level tensors have T rows per video."""
    def frames(t):
        return torch.cat([t[:ns * T], t[Bs * T:Bs * T + nt * T]]).cpu()

    def videos(t):
        return torch.cat([t[:ns], t[Bs:Bs + nt]]).cpu()
    return frames, videos


def gate_list(g):
    return [g.get("frame_disc"), *g["trn"], *g["rel_disc"], g.get("video_disc")]


def realised_gates(pool, rows_f, rows_v, kept, plain, frame_disc=True, video_disc=True):
    """The step's ReLU pattern in the oracle's gate format, and (flips, total): the units where it differs from the
    fp64 pattern ``plain`` of the same masks, of the units counted.  Shared-layer units count only where the mask
    ``kept`` keeps them (a dropped unit is 0 whatever its sign); the oracle's own sign is kept there."""
    gates = {"shared": torch.where(kept, rows_f(pool["feat"]) > 0, plain["shared"]),
             "trn": [rows_v(a) > 0 for a in pool["act"]], "rel_disc": [rows_v(h) > 0 for h in pool["hid_r"]]}
    if frame_disc:
        gates["frame_disc"] = rows_f(pool["hid_f"]) > 0
    if video_disc:
        gates["video_disc"] = rows_v(pool["hid_v"]) > 0
    flips = ((gates["shared"] != plain["shared"]) & kept).sum().item()
    total = kept.sum().item()
    for a, b in zip(gate_list(gates), gate_list(plain)):
        if a is not None:
            flips += (a != b).sum().item()
            total += a.numel()
    return gates, flips, total


def assert_dropped_units_zero(pool, rows_f, rows_v, kept, kept_v, what):
    """Shared features and ``dropped`` are zero wherever the rebuilt keep masks drop a unit.  A mask drawn with
    another seed or step leaves about half of those units nonzero."""
    assert torch.all(rows_f(pool["feat"])[~kept] == 0), f"{what}: a unit the restated mask drops is nonzero"
    assert torch.all(rows_v(pool["dropped"])[~kept_v] == 0), f"{what}: a video unit the restated mask drops is nonzero"


def assert_pinned_grads(named, g64, g32, engine, what, noise_floor=0.0):
    """Every fp64 gradient of the oracle on the pinned pattern against the step's, within PINNED_TOL plus the
    NOISE_SCALE allowance of the fp32 restatement's own error (at least ``noise_floor``).  Returns the worst
    normwise error beyond that noise."""
    from tests.test_gpu_parity import NOISE_SCALE, PINNED_TOL
    worst = 0.0
    for name, go in g64.items():
        assert named[name].grad is not None, name
        floor = max(abs_err(g32[name], go), noise_floor) * NOISE_SCALE[engine]
        assert_close(named[name].grad, go, PINNED_TOL[engine], f"{what} grad {name}", noise=floor)
        den = go.double().norm().item()
        if den > 0:
            worst = max(worst, max(0.0, abs_err(named[name].grad, go) - 8.0 * floor) / den)
    return worst
