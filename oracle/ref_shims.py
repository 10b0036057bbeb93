"""Import the UNMODIFIED reference (``/root/reference``) on CPU  --  test infrastructure.

The reference needs three environment shims to import under this image
(SURVEY.md §8c); none of them touches its arithmetic:
  1. ``colorama`` is imported at models.py:11-12 but not installed -> stub module;
  2. models.py:14 uses the bare name ``torch`` which it expected to leak from
     ``from torch.nn.init import *`` (models.py:3) -> publish it through builtins;
  3. models.py:125 builds ``torchvision.models.<base_model>(True)`` only to read
     ``fc.in_features`` (would download weights; no network) -> tiny stand-ins that
     report the pool5 width: 2048 for resnet101, 512 for resnet18 / resnet34.

``/root/reference`` exists only in the build container, never on the GPU box;
callers must check ``available()`` first.
"""
from __future__ import annotations

import builtins
import os
import sys
import types

REFERENCE_ROOT = os.environ.get("TA3N_REFERENCE_ROOT", "/root/reference")
# byte copies of models.py / TRNmodule.py / loss.py made by oracle/build_ref.py in the build container
# (git-ignored, shipped to the GPU box like a built .so) -- used where /root/reference does not exist
SNAPSHOT_ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "ta3n_ref_modules.zip")


def available() -> bool:
    """The full reference tree (models + dataset + ...) is present: build container only."""
    return os.path.isfile(os.path.join(REFERENCE_ROOT, "models.py"))


def models_root():
    """sys.path entry holding the unmodified models.py / TRNmodule.py / loss.py: the reference tree, else the
    oracle/_ref archive (zipimport), else None."""
    if all(os.path.isfile(os.path.join(REFERENCE_ROOT, f)) for f in ("models.py", "TRNmodule.py", "loss.py")):
        return REFERENCE_ROOT
    if os.path.isfile(SNAPSHOT_ROOT):
        import zipfile
        try:
            with zipfile.ZipFile(SNAPSHOT_ROOT) as z:
                if all(f in z.namelist() for f in ("models.py", "TRNmodule.py", "loss.py")):
                    return SNAPSHOT_ROOT
        except zipfile.BadZipFile:
            pass
    return None


def load():
    """Return the reference's (models, TRNmodule, loss) modules."""
    root = models_root()
    if root is None:
        raise RuntimeError(f"reference modules found neither at {REFERENCE_ROOT} nor at {SNAPSHOT_ROOT}")
    import torch
    import torchvision

    if "colorama" not in sys.modules:
        stub = types.ModuleType("colorama")

        class _Blank:
            def __getattr__(self, _name):
                return ""

        stub.init = lambda *a, **k: None
        stub.Fore, stub.Back, stub.Style = _Blank(), _Blank(), _Blank()
        sys.modules["colorama"] = stub
    builtins.torch = torch

    def head_only(width):
        fc = type("fc", (), {"in_features": width})
        return lambda *a, **k: type("HeadOnly", (), {"fc": fc})()

    for name, width in (("resnet101", 2048), ("resnet18", 512), ("resnet34", 512)):
        setattr(torchvision.models, name, head_only(width))

    if root not in sys.path:
        sys.path.insert(0, root)
    saved = {k: sys.modules.pop(k) for k in ("models", "TRNmodule", "loss") if k in sys.modules
             and not (getattr(sys.modules[k], "__file__", "") or "").startswith(root)}
    try:
        import TRNmodule as ref_trn     # noqa: E402
        import loss as ref_loss         # noqa: E402
        import models as ref_models     # noqa: E402
    finally:
        for k, v in saved.items():
            sys.modules.setdefault(k, v)
    return ref_models, ref_trn, ref_loss


def load_dataset():
    """Return the reference's `dataset` module (dataset.py needs only the colorama stub)."""
    if not available():
        raise RuntimeError(f"reference tree not found at {REFERENCE_ROOT}")
    load()                                   # installs the colorama stub and sys.path entry
    import importlib.util
    spec = importlib.util.spec_from_file_location("ta3n_reference_dataset", os.path.join(REFERENCE_ROOT, "dataset.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


import torch as _torch  # noqa: E402


class InjectedDropout(_torch.nn.Module):
    """Stand-in for the reference's ``nn.Dropout`` instances that applies a queue of
    given keep-masks (in call order) instead of drawing from the RNG, so that the
    reference and the CUDA path can be compared in train mode.  Assigned onto a
    reference *instance* (``model.dropout_i = InjectedDropout(...)``); the reference
    source is untouched."""

    def __init__(self, p, masks):
        super().__init__()
        self.p = float(p)
        self.masks = list(masks)
        self.calls = 0

    def forward(self, x):
        m = self.masks[self.calls % len(self.masks)]
        self.calls += 1
        return x * m.to(x.dtype) * (1.0 / (1.0 - self.p))
