"""Development check of the training step (GPU box): legacy and phased executors per engine vs the fp64 oracle,
per-launch and per-step timing.  python tools/step_check.py [B] [T] [C]"""
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ta3n_b200  # noqa: E402
from oracle import ta3n_oracle as orc  # noqa: E402
from ta3n_b200.models import VideoModel  # noqa: E402
from ta3n_b200.train import TrainStep  # noqa: E402

B = int(sys.argv[1]) if len(sys.argv) > 1 else 24
T = int(sys.argv[2]) if len(sys.argv) > 2 else 5
Cn = int(sys.argv[3]) if len(sys.argv) > 3 else 12
dev = torch.device("cuda:0")
cfg = orc.PathConfig(num_class=Cn, num_segments=T, fc_dim=512, dropout_i=0.0, dropout_v=0.0)
params = orc.init_params(cfg, seed=21)
g = torch.Generator().manual_seed(8)
for k in params:
    if params[k].dtype.is_floating_point and k.startswith(orc.USED_PARAM_PREFIXES) and "weight" in k:
        params[k] = params[k] + 0.02 * torch.randn(params[k].shape, generator=g)
bs, bt = B, max(B - 3, 1)
xs = torch.randn(bs, T, orc.FEATURE_DIM, generator=g)
xt = torch.randn(bt, T, orc.FEATURE_DIM, generator=g) - 0.2
labels = torch.arange(bs) % Cn
beta = (0.75, 0.6, 0.5)
p64 = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in params.items()}
l64, o64, g64 = orc.train_step(p64, xs.double(), xt.double(), labels, beta, cfg, 0.003, train=True)


def rel(a, b):
    a, b = a.detach().double().cpu().reshape(-1), b.detach().double().cpu().reshape(-1)
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def build():
    m = VideoModel(Cn, "video", "trn-m", "RGB", train_segments=T, val_segments=T, add_fc=1, fc_dim=512, dropout_i=0.0,
                   dropout_v=0.0, partial_bn=False, use_bn="none", ens_DA="none", use_attn="TransAttn",
                   use_attn_frame="none", share_params="Y", verbose=False)
    m.load_state_dict(params)
    return m.to(dev).train()


def run(mode, engine, use_graph=False):
    ta3n_b200.set_gemm_engine(engine)
    m = build()
    step = TrainStep(m, bs, bt, beta, gamma=0.003, use_graph=use_graph, mode=mode)
    loss = step(xs, xt, labels)
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.grad is not None}
    return loss.item(), grads, step, m


def report(tag, loss, grads, ref_loss, ref):
    worst = max((rel(grads[k], ref[k]), k) for k in ref)
    print(f"{tag}: loss {loss:.7f} (ref {float(ref_loss):.7f}, rel {abs(loss - float(ref_loss)) / abs(float(ref_loss)):.2e}) "
          f"worst grad {worst[0]:.2e} [{worst[1]}]", flush=True)


l_leg, g_leg, _, _ = run("legacy", "fp32")
report("legacy fp32 vs oracle", l_leg, g_leg, l64, g64)
l_x3, g_x3, _, _ = run("legacy", "tf32x3")
report("legacy tf32x3 vs oracle", l_x3, g_x3, l64, g64)
l_x3p, g_x3p, _, _ = run("phased", "tf32x3")
report("phased tf32x3 vs oracle", l_x3p, g_x3p, l64, g64)
l_ph, g_ph, _, _ = run("phased", "fp32")
report("phased fp32 vs oracle", l_ph, g_ph, l64, g64)
l_pt, g_pt, _, _ = run("phased", "tf32")
report("phased tf32 vs oracle", l_pt, g_pt, l64, g64)
# per-launch device time of the phased sequence (eager, CUDA events inside the library)
from ta3n_b200 import _lib  # noqa: E402
ta3n_b200.set_gemm_engine("tf32")
m = build()
step = TrainStep(m, bs, bt, beta, gamma=0.003, use_graph=False, mode="phased")
step.load(xs, xt, labels)
for _ in range(3):
    step.run()
_lib.timing_enable(True)
for _ in range(10):
    step.run()
torch.cuda.synchronize()
rep = _lib.timing_report()
_lib.timing_enable(False)
print("phased per launch (us):", {k: round(v[1] / 10 * 1e3, 1) for k, v in rep.items()}, flush=True)
# timing
for mode, eng in (("legacy", "tf32"), ("legacy", "tf32x3"), ("phased", "tf32"), ("phased", "tf32x3")):
    ta3n_b200.set_gemm_engine(eng)
    m = build()
    step = TrainStep(m, bs, bt, beta, gamma=0.003, use_graph=True, mode=mode)
    step.load(xs, xt, labels)
    for _ in range(5):
        step.run()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(50):
        step.run()
    b.record()
    torch.cuda.synchronize()
    print(f"{mode}/{eng}: {a.elapsed_time(b) / 50 * 1e3:.1f} us/step, launches/step {step.launches_per_step}", flush=True)
