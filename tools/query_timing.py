"""Times lb_acq_argmax_dev (UCB) for M candidates at N=16384 (panel / slab path as the library chooses).
usage: python tools/query_timing.py [M ...]"""
import ctypes as C, os, sys, numpy as np, torch
sys.path.insert(0, os.getcwd())
from limbo_b200 import _lib, kernel, mean, model, synth
N, D = 16384, 6
Ms = [int(a) for a in sys.argv[1:]] or [10000]
X = synth.points(1234, N, D); y = synth.targets(X)
st = torch.cuda.Stream(); torch.cuda.set_stream(st)
gp = model.GP(D, 1, kernel=kernel.SquaredExpARD, mean=mean.Data); gp.set_stream(st.cuda_stream)
gp.compute(X, y[:, None])
lib = _lib.load()
for M in Ms:
    Xq = synth.points(1235, M, D)
    dXq = torch.from_numpy(Xq).cuda(); dB = torch.zeros(1, dtype=torch.float64, device="cuda"); dI = torch.zeros(1, dtype=torch.int64, device="cuda")
    ap = np.array([0.5, 0.0])
    def q(): _lib.check(lib.lb_acq_argmax_dev(gp._h, 0, ap.ctypes.data, M, dXq.data_ptr(), None, float(y.mean()), None, dB.data_ptr(), dI.data_ptr()), "acq")
    for _ in range(3): q()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(5): q()
    e1.record(st); torch.cuda.synchronize()
    print("M", M, "query ms", e0.elapsed_time(e1) / 5, "best", dB.item(), dI.item())
