"""Where a slab's time goes inside the plain tensor-core GEMM kernel: per-stage clock64 stamps by warp role, from a
build of the library compiled with -DTA3N_TC_TIMELINE (off in the product build; this tool compiles it into a temporary
directory unless --lib names one already built).  Runs one full-wave launch (1408x1536, 132 tiles, K = 4096) per
operand layout through `ta3n_gemm_ex` on the plain kernel and prints, per layout, the mean over CTAs and slabs 8..63
(the ring in steady state) of each interval in cycles, and the SM clock while the kernel ran (clock64 over
globaltimer, per CTA).  Prints one JSON line.

Intervals (slab i):
  land      TMA issued -> raw stage landed, seen by the B warps (MN-major B only)
  kslot     landed -> a K-major slot free, transpose starts (MN-major B only)
  xpose     the transpose's loads and stores issued (MN-major B only)
  fence     proxy fence + ready arrival (MN-major B only)
  wait      consumers enter slab i -> A landed and B ready
  issue     ready -> A fragments loaded and the slab's MMAs issued
  retire    MMAs issued -> retired (seen at the next slab's wait_group)
  period    consumers enter slab i -> enter slab i + 1
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CTAS, SLABS, EVENTS = 132, 64, 9          # kTlCtas, kTlSlabs, kTlEvents of gemm_wgmma.cuh
TMA, FULL, XS, XE, CS, READY, REL, RET, FENCE = range(EVENTS)
M, N, K = 1408, 1536, 4096
LAYOUTS = {"KxK": (1, 1), "dgrad_KxN": (1, 0), "wgrad_MxN": (0, 0)}
FIRST = 8                                 # slabs before the ring reaches steady state


def build_instrumented(out_dir):
    from ta3n_b200 import build as b
    path = os.path.join(out_dir, "libta3n_sm90_timeline.so")
    cmd = [b._nvcc(), *b.NVCC_FLAGS, "-DTA3N_TC_TIMELINE", os.path.join(b.CSRC, "ta3n_api.cu"), "-o", path]
    subprocess.run(cmd, check=True)
    return path


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--lib", help="an instrumented libta3n_sm90 build (default: compile one into a temporary directory)")
    args = ap.parse_args()
    lib_path = args.lib or build_instrumented(tempfile.mkdtemp(prefix="ta3n_tl_"))
    os.environ["TA3N_LIB"] = lib_path

    import ctypes as C

    import numpy as np
    import torch

    import ta3n_b200
    from ta3n_b200 import _lib

    lib = _lib.load()
    read = lib.ta3n_tc_timeline_read
    read.restype, read.argtypes = C.c_int, [C.c_void_p, C.c_size_t]
    ta3n_b200.set_gemm_engine("tf32")
    dev = torch.device("cuda:0")
    buf = np.zeros(CTAS * SLABS * EVENTS + CTAS * 4, dtype=np.uint64)
    res = {"gpu": torch.cuda.get_device_name(0), "shape": f"{M}x{N}x{K}", "slabs": f"{FIRST}..{SLABS - 1}"}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        res["power_limit_w"] = float(out)
    except Exception:      # noqa: BLE001  (the timeline stands without it)
        res["power_limit_w"] = None
    for name, (ak, bk) in LAYOUTS.items():
        g = torch.Generator(device=dev).manual_seed(ak * 2 + bk)
        A = torch.randn((M, K) if ak else (K, M), device=dev, generator=g)
        B = torch.randn((N, K) if bk else (K, N), device=dev, generator=g)
        Cm = torch.empty(M, N, device=dev)
        s = torch.cuda.current_stream().cuda_stream
        for _ in range(3):       # warm-up (module load, tensor maps, clocks); the last launch is the one read
            _lib.check(lib.ta3n_gemm_ex(A.data_ptr(), K if ak else M, ak, B.data_ptr(), K if bk else N, bk,
                                        Cm.data_ptr(), N, M, N, K, None, 0, s))
            _lib.check(read(buf.ctypes.data, buf.nbytes))
        tl = buf[:CTAS * SLABS * EVENTS].reshape(CTAS, SLABS, EVENTS).astype(np.int64)
        clk = buf[CTAS * SLABS * EVENTS:].reshape(CTAS, 4).astype(np.int64)
        ghz = (clk[:, 3] - clk[:, 1]) / np.maximum(clk[:, 2] - clk[:, 0], 1)
        w = tl[:, FIRST:SLABS - 1]

        def mean(a, b, src=w):
            return round(float(np.mean(src[..., b] - src[..., a])), 1)

        r = {"sm_clock_mhz": round(float(np.median(ghz)) * 1e3, 1)}
        if not bk:
            r.update(land=mean(TMA, FULL), kslot=mean(FULL, XS), xpose=mean(XS, FENCE), fence=mean(FENCE, XE))
        r.update(wait=mean(CS, READY), issue=mean(READY, REL) if not bk else None, retire=mean(REL, RET) if not bk else None,
                 period=round(float(np.mean(tl[:, FIRST + 1:SLABS, CS] - tl[:, FIRST:SLABS - 1, CS])), 1))
        # the raw stage's whole stay in the ring, TMA issue -> released (MN-major B: max of transpose end and MMA
        # issue; K-major B: retire)
        rel = np.maximum(w[..., XE], w[..., REL]) if not bk else w[..., RET]
        r["raw_stage_held"] = round(float(np.mean(rel - w[..., TMA])), 1)
        res[name] = r
    print(json.dumps({"probe": "tc_stage_timeline", **res}))


if __name__ == "__main__":
    main()
