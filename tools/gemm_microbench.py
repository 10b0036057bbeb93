"""Time the tensor-core GEMM engine in isolation: N back-to-back launches captured in one CUDA graph."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import ta3n_b200
from ta3n_b200 import _lib
lib = _lib.load()
dev = torch.device("cuda:0")
eng = os.environ.get("ENGINE", "tf32")
ta3n_b200.set_gemm_engine(eng)
REP = 20
def bench(M, N, K, layout=(1, 1)):
    ak, bk = layout
    A = torch.randn(M, K, device=dev) if ak else torch.randn(K, M, device=dev)
    B = torch.randn(N, K, device=dev) if bk else torch.randn(K, N, device=dev)
    C = torch.empty(M, N, device=dev)
    st = torch.cuda.Stream()
    def run():
        s = torch.cuda.current_stream().cuda_stream
        for _ in range(REP):
            _lib.check(lib.ta3n_gemm_ex(A.data_ptr(), K if ak else M, ak, B.data_ptr(), K if bk else N, bk,
                                        C.data_ptr(), N, M, N, K, None, 0, s))
    with torch.cuda.stream(st):
        run()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run()
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); g.replay(); g.replay(); g.replay(); e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / (3 * REP)
    tiles = ((M + 127) // 128) * ((N + 127) // 128)
    print(f"{eng} M={M:5d} N={N:5d} K={K:5d} layout={layout} tiles={tiles:4d}  {us:8.2f} us/launch  "
          f"{2*M*N*K/us/1e6:8.1f} TFLOP/s  operand L2 traffic {tiles*K*1024/us/1e6:7.2f} TB/s")
for shape in [(128, 128, 32), (128, 128, 256), (128, 128, 2048), (512, 256, 256), (1024, 128, 256), (2560, 512, 2048),
              (2560, 512, 512), (512, 256, 2560), (18944, 1024, 1024), (8192, 8192, 1024)]:
    bench(*shape)
bench(512, 2048, 2560, (0, 0))
bench(2560, 512, 512, (1, 0))
