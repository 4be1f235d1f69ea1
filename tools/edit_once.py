"""a few steps of the BASELINE config-4 edit loop at batch 128 (a short workload for torch.profiler launch lists)"""
import importlib, os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
from oracle import weights as ow
pkg = importlib.import_module("neural-photo-editor_b200")
m = pkg.IAN("IAN_simple.py", True, weights=ow.make_simple_weights(0))
z, boxes, rgb = ow.config4_inputs(128)
zt, bt, rt = (torch.from_numpy(a).cuda() for a in (z, boxes, rgb))
torch.cuda.synchronize()
m.edit_loop_dev(zt.data_ptr(), bt.data_ptr(), rt.data_ptr(), 0, 128, int(os.environ.get("EDIT_STEPS", "3")), 0.05, 0)
torch.cuda.synchronize()
