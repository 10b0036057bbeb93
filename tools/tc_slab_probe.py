"""Per-slab cost of the plain tensor-core GEMM kernel in each operand layout, through `ta3n_gemm_ex` at K = 4096 and
8192: the slope of the time per launch over the 128 extra 32-wide K slabs, in cycles at the SM clock read in the same
run under load (sampled while the full-wave K x K graph replays).  Two grids: one 128x128 output tile (one CTA alone on the GPU) and one full wave (1408x1536, 132 tiles: every SM
of an H100 SXM busy, as in the training step's large launches).  Prints one JSON line."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import ta3n_b200  # noqa: E402
from ta3n_b200 import _lib  # noqa: E402

GRIDS = {"tile": (128, 128), "wave": (1408, 1536)}
LAYOUTS = {"KxK": (1, 1), "dgrad_KxN": (1, 0), "wgrad_MxN": (0, 0), "MxK": (0, 1)}
KS = (4096, 8192)
REP, ROUNDS = 50, 7


def gpu_facts():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, pl, sm, smax = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit_w": float(pl), "sm_clock_mhz_idle": float(sm), "sm_clock_max_mhz": float(smax)}
    except Exception as e:     # noqa: BLE001  (the timings stand without it)
        return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi_error": str(e)}


def loaded_sm_clock(graph, seconds=1.0):
    """clocks.sm read by nvidia-smi while `graph` replays back to back for about `seconds`."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    graph.replay()
    e1.record()
    torch.cuda.synchronize()
    for _ in range(max(1, int(seconds * 1e3 / e0.elapsed_time(e1)))):
        graph.replay()
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        mhz = float(out)
    except Exception:      # noqa: BLE001
        mhz = None
    torch.cuda.synchronize()
    return mhz


def graph_of(lib, M, N, K, ak, bk, dev):
    g = torch.Generator(device=dev).manual_seed(K + 2 * ak + bk)
    A = torch.randn((M, K) if ak else (K, M), device=dev, generator=g)
    B = torch.randn((N, K) if bk else (K, N), device=dev, generator=g)
    C = torch.empty(M, N, device=dev)

    def run():
        s = torch.cuda.current_stream().cuda_stream
        for _ in range(REP):
            _lib.check(lib.ta3n_gemm_ex(A.data_ptr(), K if ak else M, ak, B.data_ptr(), K if bk else N, bk,
                                        C.data_ptr(), N, M, N, K, None, 0, s))

    side = torch.cuda.Stream()
    with torch.cuda.stream(side):          # warm-up: module load and tensor-map encoding outside the capture
        run()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run()
    graph.replay()
    torch.cuda.synchronize()
    graph.keep = (A, B, C)
    return graph


def us_per_launch(graph):
    times = []
    for _ in range(ROUNDS):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        graph.replay()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1e3 / REP)
    return sorted(times)[ROUNDS // 2]


def main():
    dev = torch.device("cuda:0")
    ta3n_b200.set_gemm_engine("tf32")       # every launch on the plain kernel
    lib = _lib.load()
    facts = gpu_facts()
    res, graphs = {}, {}
    for grid, (M, N) in GRIDS.items():
        for name, (ak, bk) in LAYOUTS.items():
            for K in KS:
                graphs[grid, name, K] = graph_of(lib, M, N, K, ak, bk, dev)
    facts["sm_clock_mhz_under_load"] = loaded_sm_clock(graphs["wave", "KxK", KS[1]])
    mhz = facts["sm_clock_mhz_under_load"] or facts.get("sm_clock_max_mhz", 1980.0)
    for grid, (M, N) in GRIDS.items():
        for name, (ak, bk) in LAYOUTS.items():
            t = {K: us_per_launch(graphs[grid, name, K]) for K in KS}
            slope_us = (t[KS[1]] - t[KS[0]]) / ((KS[1] - KS[0]) // 32)
            res[f"{grid}/{name}"] = {"us_per_launch": {str(K): round(v, 3) for K, v in t.items()},
                                     "us_per_slab": round(slope_us, 5), "cycles_per_slab": round(slope_us * mhz, 1)}
    print(json.dumps({"probe": "tc_slab", "grids": {k: f"{m}x{n}" for k, (m, n) in GRIDS.items()}, "k": list(KS),
                      "clock_for_cycles_mhz": mhz, **facts, "layouts": res}))


if __name__ == "__main__":
    main()
