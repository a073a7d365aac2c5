"""Fresh process: two forwards of the sparse decoder, every libwmd op's outputs compared between them (the first forward
runs every kernel cold: timing-dependent races show up as differences)."""
import os, sys; sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from wavelet_monodepth_b200 import kitti_decoders as kd, ops, synth
DEV = 'cuda'
ch = synth.RESNET18_CH if len(sys.argv) < 2 or sys.argv[1] == "r18" else synth.RESNET50_CH
hw = (192, 640) if ch == synth.RESNET18_CH else (320, 1024)
nb = 16 if ch == synth.RESNET18_CH else 8
mod = kd.SparseDepthWaveProgressiveDecoder(np.array(ch)); synth.load_random(mod, seed=1, gains={".2.conv.": 4.0})
feats = [torch.rand(s, device=DEV, generator=torch.Generator(DEV).manual_seed(3 + i)) for i, s in enumerate(synth.kitti_feature_shapes(nb, *hw, ch))]
mod = mod.to(DEV).eval()
log = {}
def wrap(name):
    real = getattr(ops, name)
    def f(*a, **k):
        r = real(*a, **k)
        vals = list(r.values()) if isinstance(r, dict) else (list(r) if isinstance(r, tuple) else [r])
        extra = ""
        if name == "conv_rows":
            extra = " taps%d c%s+%s->%d count=%s" % (k.get("taps", 9), a[1], k.get("c1", 0), a[4], "dev" if k.get("count") is not None else "-")
            cnt = k.get("count")
        log[cur].append((name + extra, [v for v in vals if torch.is_tensor(v)], k.get("count") if name in ("conv_rows", "head_mlp") else None, a[4] if name == "conv_rows" else None))
        return r
    setattr(ops, name, f)
for nm in ("conv_rows", "head_gather", "head_idwt", "head_mlp", "nchw_to_rows", "level_masks", "compact", "gate_map"):
    wrap(nm)
for rep in range(3):
    cur = rep; log[cur] = []
    out = mod(feats, 0.05)
    torch.cuda.synchronize()
    log[cur] = [(n, [t.clone() for t in ts], (int(c[0]) if c is not None else None), co) for n, ts, c, co in log[cur]]
for other in (1, 2):
    print("forward 0 vs forward %d" % other)
    for k, ((na, ta, ca, co), (nb_, tb, cb, _)) in enumerate(zip(log[0], log[other])):
        res = []
        for x, y in zip(ta, tb):
            if x.shape != y.shape:
                res.append("shape"); continue
            if x.dtype == torch.float32 and x.dim() == 2 and co is not None:        # conv rows: only valid rows / columns
                rows = ca if ca is not None else x.shape[0]
                x, y = x[:rows, :co], y[:rows, :co]
            elif x.dtype == torch.float32 and x.dim() == 2 and ca is not None:
                x, y = x[:ca, :54], y[:ca, :54]
            d = (x.float() - y.float()).abs()
            nbad = int((d > 0).sum())
            res.append("ok" if nbad == 0 else "DIFF n=%d max=%.3g rows=%s" % (nbad, float(d.max()), sorted(set((d > 0).nonzero()[:, 0].tolist()))[:6]))
        if any(r != "ok" for r in res):
            print("  ", k, na, res)
print("done")
