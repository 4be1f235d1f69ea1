"""run the full-IAN reconstruct a few times at batch 512 (a short workload for torch.profiler launch lists)"""
import importlib, os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
from oracle import weights as ow
pkg = importlib.import_module("neural-photo-editor_b200")
m = pkg.IAN("IAN.py", True, weights=ow.make_full_weights(0))
if os.environ.get("FULL_PREC"):
    m.set_precision(os.environ["FULL_PREC"])
n = int(os.environ.get("FULL_N", "512"))
x = torch.from_numpy(np.random.default_rng(0).uniform(-1, 1, (n, 3, 64, 64)).astype(np.float32)).cuda()
z = torch.empty(n, 100, device="cuda"); xh = torch.empty(n, 3, 64, 64, device="cuda")
torch.cuda.synchronize()
for _ in range(int(os.environ.get("FULL_IT", "3"))):
    m.reconstruct_dev(x.data_ptr(), n, z.data_ptr(), xh.data_ptr(), 0)
torch.cuda.synchronize()
