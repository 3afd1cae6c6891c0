import sys, time
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import torch
import __graft_entry__ as ge
pkg = ge.load_package()
ft = pkg.FtSgemm()
n = 256
dA = torch.randn(n*n, device='cuda'); dB = torch.randn(n*n, device='cuda'); dC = torch.zeros(n*n, device='cuda')
stream = torch.cuda.current_stream().cuda_stream
opts = pkg.make_opts(stream=stream)
for kid in (7, 3, 21, 13, 31):
    for _ in range(20): ft.run(kid, n, n, n, dA, dB, dC, 1.0, 0.0, opts)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(2000): ft.run(kid, n, n, n, dA, dB, dC, 1.0, 0.0, opts)
    t1 = time.perf_counter()
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    print(kid, 'enqueue us/call', round((t1-t0)/2000*1e6, 2), 'total us/call', round((t2-t0)/2000*1e6, 2), flush=True)
