import os, sys; sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, torch.nn.functional as F
from wavelet_monodepth_b200 import ops
dev = 'cuda'
torch.manual_seed(0)
for (n, c, h, w, dens) in ((32, 64, 160, 512, 0.163), (32, 256, 80, 256, 0.283), (32, 512, 40, 128, 0.498)):
    x = torch.rand(n, c, h, w, device=dev)
    seeds = (torch.rand(n, 1, h // 8, w // 8, device=dev) < dens * 0.55).float()
    m = F.interpolate(seeds, scale_factor=8, mode="nearest")
    m = F.max_pool2d(m, 5, 1, 2).to(torch.uint8)
    _, pix, off = ops.compact(m, want_idxmap=False)
    cnt = int(off[n])
    def t(fn, reps=5):
        fn(); torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps): fn()
        e1.record(); torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps * 1e3
    tg = t(lambda: ops.gather_rows_list(x, pix, off[n:]))
    td = t(lambda: ops.nchw_to_rows(x))
    mb = cnt * c * 8 / 1e6
    print("c %d grid %dx%d density %.3f: list gather %.1f us (%.0f MB -> %.2f TB/s), dense move %.1f us" % (c, h, w, cnt / (n * h * w), tg, mb, mb / tg / 1e6 * 1e6 / 1e6, td))
