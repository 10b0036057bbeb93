import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, ta3n_b200
from ta3n_b200 import _lib
lib = _lib.load(); dev = torch.device("cuda:0"); ta3n_b200.set_gemm_engine("tf32")
REP = 20
for (M, N, K) in [(128, 128, 32), (512, 256, 256)]:
    A = torch.randn(M, K, device=dev); B = torch.randn(N, K, device=dev); C = torch.empty(M, N, device=dev)
    def run():
        s = torch.cuda.current_stream().cuda_stream
        for _ in range(REP):
            _lib.check(lib.ta3n_gemm_ex(A.data_ptr(), K, 1, B.data_ptr(), K, 1, C.data_ptr(), N, M, N, K, None, 0, s))
    st = torch.cuda.Stream()
    with torch.cuda.stream(st): run()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g): run()
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); g.replay(); g.replay(); e1.record(); torch.cuda.synchronize()
    print(f"M={M} N={N} K={K}: {e0.elapsed_time(e1)*1e3/(2*REP):7.2f} us/launch")
