"""Generate ``tests/golden/eval_golden.npz``: ``validate()`` of the UNMODIFIED reference (main.py:669-761).

Run in the build container only (needs /root/reference):

    python -m oracle.gen_golden_eval

Per case the reference ``VideoModel`` (seeded init, every weight then moved by 0.02 N(0,1), as gen_golden_mcd does, so
that the predictions spread over the classes) runs in ``eval()`` under ``no_grad`` exactly as main.py:707 calls it --
``model(val, val, [0]*3, 0, is_train=False, reverse=False)`` on batches of ``batch`` rows, the last one zero-padded
(main.py:690-693) -- then ``removeDummy`` (:710), ``CrossEntropyLoss(weight=...)`` (:205, :725) and ``accuracy``
(:726).  ``accuracy`` and ``removeDummy`` are taken from main.py by ``ast`` at generation time; nothing of main.py is
stored.  Stored per case: the labels and class weights, the target-half logits and attention of every row, the
per-batch loss / prec@1 / prec@5, the epoch averages (AverageMeter, :728-730) and |fp32 - fp64| of the reference's
logits and attention (the noise floor).
"""
from __future__ import annotations

import ast
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import ref_shims  # noqa: E402
from oracle import ta3n_oracle as orc  # noqa: E402
from oracle.gen_golden_mcd import perturb  # noqa: E402

GOLDEN_PATH = os.path.join(os.path.dirname(HERE), "tests", "golden", "eval_golden.npz")
CASES = {
    # name: dict(agg, T (train_segments), Tv (val_segments), C, F, use_attn, attn_frame, ens, N, batch, weighted)
    "transattn_T5": dict(agg="trn-m", T=5, Tv=5, C=8, F=256, use_attn="TransAttn", attn_frame="none", ens="none",
                         N=21, batch=8, weighted=False),
    "transattn_T5_w": dict(agg="trn-m", T=5, Tv=5, C=8, F=256, use_attn="TransAttn", attn_frame="none", ens="none",
                           N=21, batch=8, weighted=True),
    "none": dict(agg="trn-m", T=5, Tv=5, C=6, F=128, use_attn="none", attn_frame="none", ens="none", N=13, batch=5,
                 weighted=True),
    "general": dict(agg="trn-m", T=5, Tv=5, C=7, F=128, use_attn="general", attn_frame="none", ens="none", N=11,
                    batch=4, weighted=False),
    "attnframe_T4": dict(agg="trn-m", T=4, Tv=4, C=9, F=128, use_attn="TransAttn", attn_frame="TransAttn", ens="none",
                         N=10, batch=4, weighted=True),
    "avgpool_Tv7": dict(agg="avgpool", T=5, Tv=7, C=6, F=256, use_attn="TransAttn", attn_frame="none", ens="none",
                        N=12, batch=5, weighted=False),
    "avgpool_none_Tv3": dict(agg="avgpool", T=5, Tv=3, C=5, F=128, use_attn="none", attn_frame="none", ens="none",
                             N=9, batch=4, weighted=True),
    "mcd": dict(agg="trn-m", T=5, Tv=5, C=10, F=128, use_attn="TransAttn", attn_frame="none", ens="MCD", N=9,
                batch=4, weighted=True),
}
MODEL_SEED, PERTURB_SEED, INPUT_SEED = 41, 42, 43


def case_config(c) -> orc.PathConfig:
    return orc.PathConfig(num_class=c["C"], num_segments=c["T"], fc_dim=c["F"], dropout_i=0.5, dropout_v=0.5,
                          use_attn=c["use_attn"], use_attn_frame=c["attn_frame"], ens_DA=c["ens"],
                          frame_aggregation=c["agg"])


def case_inputs(c):
    """(x [N, Tv, 2048], labels [N], class weights [C] or None) -- shared by the generator and the tests."""
    g = torch.Generator().manual_seed(INPUT_SEED)
    x = torch.randn(c["N"], c["Tv"], orc.FEATURE_DIM, generator=g)
    labels = torch.randint(0, c["C"], (c["N"],), generator=g)
    weight = (0.5 + torch.rand(c["C"], generator=g)) if c["weighted"] else None
    return x, labels, weight


def case_params(c, order):
    """The reference model's parameters (state_dict) of a case: seeded init, then the perturbation in ``order``."""
    params = orc.init_params(case_config(c), seed=MODEL_SEED)
    perturb(params, order, PERTURB_SEED)
    return params


class _ViewToReshape(ast.NodeTransformer):
    """``accuracy`` calls ``correct[:k].view(-1)`` on the transposed (non-contiguous) top-k mask, which the torch of
    its time accepted and current torch rejects; ``reshape(-1)`` gives the same values (a copy instead of a view)."""

    def visit_Attribute(self, node):
        self.generic_visit(node)
        if node.attr == "view":
            node.attr = "reshape"
        return node


def main_py_functions(names=("accuracy", "removeDummy")):
    """The named top-level functions of the reference's main.py, compiled from its source (not imported: main.py
    parses arguments at import).  In ``accuracy``, ``.view`` runs as ``.reshape`` (see _ViewToReshape)."""
    path = os.path.join(ref_shims.REFERENCE_ROOT, "main.py")
    tree = ast.parse(open(path).read(), path)
    body = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in names]
    body = [_ViewToReshape().visit(n) if n.name == "accuracy" else n for n in body]
    mod = ast.Module(body=body, type_ignores=[])
    ns = {"torch": torch}
    exec(compile(mod, path, "exec"), ns)
    return [ns[n] for n in names]


def run_reference(c, dtype=torch.float32):
    ref_models, _, _ = ref_shims.load()
    accuracy, removeDummy = main_py_functions()
    x, labels, weight = case_inputs(c)
    x = x.to(dtype)
    torch.manual_seed(MODEL_SEED)
    model = ref_models.VideoModel(c["C"], "video", c["agg"], "RGB", train_segments=c["T"], val_segments=c["Tv"],
                                  add_fc=1, fc_dim=c["F"], dropout_i=0.5, dropout_v=0.5, partial_bn=False,
                                  use_bn="none", ens_DA=c["ens"], use_attn=c["use_attn"], n_attn=1,
                                  use_attn_frame=c["attn_frame"], share_params="Y", verbose=False).to(dtype)
    order = [k for k, _ in model.named_parameters()]
    perturb(dict(model.named_parameters()), order, PERTURB_SEED)
    model.eval()
    criterion = torch.nn.CrossEntropyLoss(weight=None if weight is None else weight.to(dtype))
    B = c["batch"]
    outs, attns, per_batch = [], [], []
    with torch.no_grad():
        for a in range(0, c["N"], B):
            val_data, val_label = x[a:a + B], labels[a:a + B]
            n = val_data.size(0)
            if n < B:                                                                          # main.py:690-693
                val_data = torch.cat((val_data, torch.zeros(B - n, val_data.size(1), val_data.size(2), dtype=dtype)))
            _, _, _, _, _, attn_val, out_val, out_val_2, pred_domain_val, feat_val = \
                model(val_data, val_data, [0] * 3, 0, is_train=False, reverse=False)          # main.py:707
            attn_val, out_val, out_val_2, pred_domain_val, feat_val = \
                removeDummy(attn_val, out_val, out_val_2, pred_domain_val, feat_val, n)         # main.py:710
            loss = criterion(out_val, val_label)
            prec1, prec5 = accuracy(out_val.data, val_label, topk=(1, 5))
            per_batch.append((loss.item(), prec1.item(), prec5.item(), out_val.size(0)))
            outs.append(out_val)
            attns.append(attn_val.reshape(n, -1))
    return order, torch.cat(outs), torch.cat(attns), per_batch


def main():
    blob = {}
    meta = {"seeds": [MODEL_SEED, PERTURB_SEED, INPUT_SEED], "cases": CASES, "torch": torch.__version__}
    for name, c in CASES.items():
        order, logits, attn, per_batch = run_reference(c)
        _, logits64, attn64, _ = run_reference(c, torch.float64)
        x, labels, weight = case_inputs(c)
        k = name + "/"
        blob[k + "labels"] = labels.numpy()
        if weight is not None:
            blob[k + "class_weight"] = weight.double().numpy()
        blob[k + "logits"] = logits.double().numpy()
        blob[k + "attn"] = attn.double().numpy()
        blob[k + "noise/logits"] = np.array((logits.double() - logits64).norm().item())
        blob[k + "noise/attn"] = np.array((attn.double() - attn64).norm().item())
        pb = np.array(per_batch, dtype=np.float64)          # loss, prec1, prec5, n per batch
        blob[k + "batch"] = pb
        n = pb[:, 3].sum()
        blob[k + "epoch"] = np.array([(pb[:, 0] * pb[:, 3]).sum() / n, (pb[:, 1] * pb[:, 3]).sum() / n,
                                      (pb[:, 2] * pb[:, 3]).sum() / n])        # AverageMeter avg, main.py:728-730
        meta[k + "param_order"] = order
        print(f"{name}: loss={blob[k + 'epoch'][0]:.6f} prec1={blob[k + 'epoch'][1]:.2f} "
              f"prec5={blob[k + 'epoch'][2]:.2f} noise={float(blob[k + 'noise/logits']):.2e}")
    blob["meta_json"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(GOLDEN_PATH, **blob)
    print("wrote", GOLDEN_PATH, os.path.getsize(GOLDEN_PATH), "bytes")


if __name__ == "__main__":
    main()
