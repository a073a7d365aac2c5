import os, sys; sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from wavelet_monodepth_b200 import ops
from wavelet_monodepth_b200._lib import PAD_REFLECT, ACT_ELU
torch.manual_seed(0)
dev='cuda'
for (n,h,w,cin,cout) in ((1,6,20,512,256),(1,12,40,512,256),(1,12,40,256,576),(16,6,20,512,256)):
    x = torch.rand(n*h*w, cin, device=dev)
    wt = (torch.rand(cout, cin, 3, 3, device=dev)-0.5)*0.05
    b = torch.rand(cout, device=dev)
    wp = ops.pack_weight(wt, 0, kind="tc")
    ref = ops.conv_rows(x, cin, wp, b, cout, n, h, w, pad=PAD_REFLECT, act=ACT_ELU, splits=1).clone()
    outs = [ops.conv_rows(x, cin, wp, b, cout, n, h, w, pad=PAD_REFLECT, act=ACT_ELU, splits=0).clone() for _ in range(4)]
    torch.cuda.synchronize()
    for k,o in enumerate(outs):
        d = (o-ref).abs()
        bad = (d > 1e-4*ref.abs().max()).nonzero()
        print((n,h,w,cin,cout), "run", k, "max diff", float(d.max()), "bad", bad.shape[0], "equal to run0", torch.equal(o, outs[0]),
              "bad rows", sorted(set((bad[:,0]//256).tolist()))[:10], "bad cols", sorted(set((bad[:,1]//32).tolist()))[:10])
# 1x1 stages at small row counts (tiled TMA loads past the last row)
for rows, cin, cout in ((480, 576, 63), (480, 256, 576), (120, 64, 54), (1920, 128, 256)):
    t = torch.rand(rows, cin, device=dev)
    wt = (torch.rand(cout, cin, 1, 1, device=dev) - 0.5)
    ref = (t.double() @ wt.reshape(cout, cin).double().t())
    wp = ops.pack_weight(wt, 0, kind="tc")
    z = ops.conv_rows(t, cin, wp, None, cout, 1, 1, rows, taps=1)
    d = (z[:, :cout].double() - ref).abs()
    print("1x1", rows, cin, cout, "max diff", float(d.max()), "bad rows", sorted(set((d > 1e-3).nonzero()[:, 0].tolist()))[:8])
