"""Per-layer CUDA-event times of one bench step (A/B of builds: run it once per library, WMD_LIB_PATH selects it)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from wavelet_monodepth_b200 import _lib
if os.environ.get('WMD_LIB_PATH'):
    _lib.LIB_PATH = os.path.abspath(os.environ['WMD_LIB_PATH'])
import bench
from wavelet_monodepth_b200 import ops
from wavelet_monodepth_b200.kitti_decoders import SparseDepthWaveProgressiveDecoder
wl = bench.WORKLOADS[bench.MAIN]
dec = SparseDepthWaveProgressiveDecoder(np.array(wl["ch"])); bench.synth_params(dec); dec = dec.cuda().eval()
feats = [f.cuda() for f in bench.synth_features(wl, wl["per_gpu_batch"], 0, pin=False)]
dec(feats, bench.THRESH)
prof = ops.Profiler(); torch.cuda.synchronize(); ops.set_profiler(prof)
for _ in range(3):
    dec(feats, bench.THRESH)
torch.cuda.synchronize(); ops.set_profiler(None)
tab = bench.conv_layer_table(prof.results(), 6570.9, 761.6, 3)
print("sum %.1f us" % sum(l["us"] for l in tab))
print("  " + "  ".join("%s%s->%d:%.0f" % (l["taps"], l["cin"], l["cout"], l["us"]) for l in tab))
