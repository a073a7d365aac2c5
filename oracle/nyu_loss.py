"""numpy fp64 restatement of NYUv2's supervised training loss as libwmd computes it (include/wmd_loss.h), with its
gather adjoint, and the seeded cases oracle/pin_nyu_loss.py runs the reference on.

The reference (NYUv2/train.py:279-327) upsamples each ("disp", s) by F.interpolate(scale_factor=2**s, mode="bilinear",
align_corners=True) and takes nn.L1Loss against the target.  The contract keeps torch's fp32 source index and lambda
(UpSample.h: area_pixel_compute_scale, compute_source_index_and_lambda) but takes 1 - lambda exactly in fp64 and the
sample in fp64 from the fp32 inputs.  numpy's fp64 operations round like the device's _rn intrinsics, and the
expressions below keep the device's order, so samples, signs and gradients are the device's bits; the means are fp64
sums in numpy's order, so they may differ from the device's by one fp32 rounding.
"""
import numpy as np

SCALES = (0, 1, 2, 3)


def axis_taps(n_in, n_out, weights="fp32"):
    """torch's align_corners taps of one axis -> (i0, i1, l0, l1).  weights="fp32" is the contract: l1 the fp32 lambda,
    l0 = 1 - l1 in fp64.  weights="fp64" is torch's rule for a float64 tensor (scale, source index, lambda and 1 - lambda
    all fp64), which the reference's float64 run uses: the oracle's adjoint in that mode is checked against it."""
    dt = np.float32 if weights == "fp32" else np.float64
    r = dt(n_in - 1) / dt(n_out - 1) if n_out > 1 else dt(0)
    src = dt(r) * np.arange(n_out, dtype=dt)
    i0 = np.minimum(src.astype(np.int64), n_in - 1)
    i1 = i0 + (i0 < n_in - 1)
    l1 = np.clip(src - i0.astype(dt), dt(0), dt(1)).astype(np.float64)
    return i0, i1, 1.0 - l1, l1


def upsample(pred, H, W, weights="fp32"):
    """(N, h, w) fp32 -> (N, H, W) fp64: l0y (l0x a + l1x b) + l1y (l0x c + l1x d), every tap read and multiplied
    (factor 1 is the identity)."""
    p = np.asarray(pred, np.float32).astype(np.float64)
    if p.shape[1:] == (H, W):
        return p                                           # factor 1: the identity, no neighbour is read
    iy0, iy1, ly0, ly1 = axis_taps(p.shape[1], H, weights)
    ix0, ix1, lx0, lx1 = axis_taps(p.shape[2], W, weights)
    r0, r1 = p[:, iy0], p[:, iy1]
    top = lx0 * r0[:, :, ix0] + lx1 * r0[:, :, ix1]
    bot = lx0 * r1[:, :, ix0] + lx1 * r1[:, :, ix1]
    return ly0[:, None] * top + ly1[:, None] * bot


def signs(sample, target):
    """sgn(sample - t) of the fp64 difference: 0 on an exact tie and on NaN."""
    d = sample - np.asarray(target).astype(np.float64)
    return (d > 0).astype(np.int8) - (d < 0).astype(np.int8)


def term(pred, target, weights="fp32"):
    """mean |upsample(pred) - t| in fp64, rounded once to fp32 (NaN for N = 0, as torch's mean of nothing).  The target
    is fp32 in the contract; an fp64 one (the reference's float64 run) is taken as it is."""
    t = np.asarray(target)
    s = upsample(pred, t.shape[1], t.shape[2], weights)
    with np.errstate(invalid="ignore"):
        return np.float32(np.abs(s - t.astype(np.float64)).sum() / t.size)


def adjoint_matrix(n_in, n_out, weights="fp32"):
    """(n_out, n_in) fp64: row d holds destination d's weights (l0 at i0, l1 at i1, l0 + l1 when they coincide)."""
    i0, i1, l0, l1 = axis_taps(n_in, n_out, weights)
    a = np.zeros((n_out, n_in))
    rows = np.arange(n_out)
    a[rows, i0] = l0
    a[rows, i1] += l1
    return a


def adjoint(sg, h, w, weights="fp32"):
    """The gather adjoint: (N, H, W) signs -> (N, h, w) fp64 S = sum over Y ascending of wy (sum over X of s wx).  The
    inner sums are exact (the weights are multiples of 2^-27 and few), so a matrix product gives their bits; the outer
    one is accumulated in ascending Y, as the device does (it skips the Y outside a pixel's footprint, where this adds
    an exact zero)."""
    sg = np.asarray(sg, np.float64)
    ay, ax = adjoint_matrix(h, sg.shape[1], weights), adjoint_matrix(w, sg.shape[2], weights)
    q = sg @ ax                                            # (N, H, w), exact
    acc = np.zeros((sg.shape[0], h, w))
    for Y in range(sg.shape[1]):
        acc = acc + ay[Y][None, :, None] * q[:, Y][:, None, :]
    return acc


def grad(pred, target, g, weights="fp32"):
    """d term / d pred for upstream gradient g (the device reads an fp32 one): fp32((g / (N H W)) S)."""
    t = np.asarray(target)
    sg = signs(upsample(pred, t.shape[1], t.shape[2], weights), t)
    coef = np.float64(g) / np.float64(t.size)
    return (coef * adjoint(sg, pred.shape[1], pred.shape[2], weights)).astype(np.float32)


def losses(preds, target, ll=None, ll_target=None, loss_scales=SCALES, supervise_ll=False, weights="fp32"):
    """The reference's dictionary from the terms: preds {s: (N, h, w)} and target (N, H, W); ll / ll_target optional.
    Scalar arithmetic in float32, in train.py's order."""
    out, total = {}, np.float32(0)
    for s in sorted(preds):
        l_depth = term(preds[s], target, weights)
        loss = np.float32(np.float32(0.1) * l_depth)
        if s in loss_scales:
            total = np.float32(total + loss)
        out["loss/%d" % s], out["loss_depth/%d" % s] = loss, l_depth
    if ll is not None:
        l_ll = np.float32(term(ll, ll_target, weights) / np.float32(16))
        out["loss_LL3"] = l_ll
        if supervise_ll:
            total = np.float32(total + l_ll)
    out["loss"] = total
    return out


# ---------------------------------------------------------------------------------------------- seeded cases
# name -> (N, H, W, disparity, use_wavelets, supervise_LL, kind).  240 x 320 is DecoderWave's pyramid (its LL is
# ("wavelets", 2, "LL"), so no LL term), 224 x 224 DecoderWave224's with its 14 x 14 LL; "thin" has a 1-pixel-wide
# coarsest scale.
CASES = {
    "d240": (2, 240, 320, False, False, False, "random"),
    "d240_disp": (2, 240, 320, True, False, False, "random"),
    "w224_disp": (2, 224, 224, True, True, False, "random"),
    "w224_sLL": (2, 224, 224, False, True, True, "random"),
    "ties": (1, 240, 320, False, False, False, "ties"),
    "nan": (2, 224, 224, True, True, True, "nan"),
    "thin": (2, 24, 8, False, False, False, "random"),
}


def case_inputs(name, seed):
    """-> depth (N, 1, H, W) float32 in [10, 1000] (the loader's clamp), preds {s: (N, 1, H/2^s, W/2^s)} float32 and
    ll (N, 1, H/16, W/16) float32 or None.  Predictions are the target (10 / depth with disparity, as torch computes it:
    reciprocal then times 10, in float32) plus noise at their own resolution, so the differences change sign often.
    "ties": the prediction is one constant at every scale and the target equals it exactly on the left half of the
    frame.  "nan": one NaN in ("disp", 1) of frame 0 and one in the LL of frame 1."""
    n, H, W, disparity, use_wavelets, _, kind = CASES[name]
    rng = np.random.default_rng(seed)
    depth = rng.uniform(10.0, 1000.0, (n, 1, H, W)).astype(np.float32)
    if kind == "ties":
        c = np.float32(250.0)
        depth[..., :W // 2] = c
        preds = {s: np.full((n, 1, H >> s, W >> s), c, np.float32) for s in SCALES}
        return depth, preds, None
    tgt = (np.float32(1) / depth * np.float32(10)).astype(np.float32) if disparity else depth
    preds = {}
    for s in SCALES:
        base = tgt[..., ::1 << s, ::1 << s]
        preds[s] = (base * rng.uniform(0.7, 1.3, base.shape)).astype(np.float32)
    ll = None
    if use_wavelets:
        base = tgt.reshape(n, 1, H // 16, 16, W // 16, 16).mean(axis=(3, 5)) * 16
        ll = (base * rng.uniform(0.7, 1.3, base.shape)).astype(np.float32)
    if kind == "nan":
        preds[1][0, 0, 5, 7] = np.nan
        ll[1, 0, 3, 4] = np.nan
    return depth, preds, ll
