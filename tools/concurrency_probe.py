"""Do two independent sub-wave tensor-core GEMM launches overlap when captured on forked streams?"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, ta3n_b200
from ta3n_b200 import _lib
lib = _lib.load(); dev = torch.device("cuda:0"); ta3n_b200.set_gemm_engine("tf32")
M, N, K = 2560, 512, 2048     # 80 tiles
A = [torch.randn(M, K, device=dev) for _ in range(2)]
B = [torch.randn(N, K, device=dev) for _ in range(2)]
C = [torch.empty(M, N, device=dev) for _ in range(2)]
def gemm(i, stream):
    _lib.check(lib.ta3n_gemm_ex(A[i].data_ptr(), K, 1, B[i].data_ptr(), K, 1, C[i].data_ptr(), N, M, N, K, None, 0, stream))
side = torch.cuda.Stream()
def seq():
    s = torch.cuda.current_stream().cuda_stream
    for _ in range(10):
        gemm(0, s); gemm(1, s)
def par():
    main = torch.cuda.current_stream()
    for _ in range(10):
        e = torch.cuda.Event(); e.record(main); side.wait_event(e)
        gemm(0, main.cuda_stream); gemm(1, side.cuda_stream)
        main.wait_stream(side)
for name, fn in (("sequential", seq), ("forked", par)):
    st = torch.cuda.Stream()
    with torch.cuda.stream(st): fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g): fn()
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); g.replay(); g.replay(); e1.record(); torch.cuda.synchronize()
    print(f"PDL={os.environ.get('TA3N_PDL','1')} {name:10s}: {e0.elapsed_time(e1)*1e3/20:7.2f} us per pair of 80-tile GEMMs")
