"""numpy restatement of KITTI's stereo depth-hints training loss, the contract of include/wmd_loss_kitti.h.

The objective is the reference's ``Trainer.generate_images_pred`` + ``Trainer.compute_losses_hints``
(KITTI/trainer.py:329-560) for ``--use_depth_hints --frame_ids 0 --use_stereo``: the only source frame is the stereo
pair, automasking and SSIM are on, ``v1_multiscale`` and ``avg_reprojection`` are off.

Two modes:
  * ``contract``: the device's fp32 rounding points (the warped colours, the three per-pixel losses before the argmin,
    the noise term, the reported terms); everything else in fp64 with the device's operation order, so the device's
    bits are expected within one fp32 ulp of this (sums differ from the device's in order only);
  * ``fp64``: no rounding point at all but the reference's own (its float32 mask counts: ``_count``), to hold the
    hand-written adjoint to torch autograd of the float64 reference.

``run(...)`` returns the terms, the warped colours, the masks and (optionally) the gradient of the total with respect to
each ("disp", s).  The adjoint is the same gather the device computes: per-centre SSIM coefficients, a 3x3 gather over
the reflected windows, the bilinear sample's derivative in its coordinates (0 where the border clamp is active, and at a
coordinate exactly on the border), the projection's closed-form derivative in depth, disp_to_depth, the upsample's
adjoint and the smoothness term with its per-frame mean.
"""
import os

import numpy as np

SCALES = (0, 1, 2, 3)
C1, C2 = 0.01 ** 2, 0.03 ** 2
PROJ_EPS = 1e-7
MASK_EPS = 1e-7
NOISE_SCALE = np.float32(1e-5)
HINT_PENALTY = np.float32(1000.0)
W_SSIM, W_L1 = 0.85, 0.15

f64, f32 = np.float64, np.float32


def _r32(x, contract):
    return x.astype(f32).astype(f64) if contract else x


def _count(m, contract):
    """a masked mean's denominator, mask count + 1e-7: fp64 on the device (contract); in the reference the masks are
    float32 even in its float64 run, so the count and its + 1e-7 are float32, where 1e-7 rounds away from a count >= 1"""
    return m + MASK_EPS if contract else float(f32(m) + f32(MASK_EPS))


def _axis_taps(n_in, n_out):
    """torch's align_corners=False source taps per destination index (exact at power-of-two factors)"""
    d = np.arange(n_out, dtype=f64)
    src = np.maximum((d + 0.5) * (n_in / n_out) - 0.5, 0.0)
    i0 = np.floor(src).astype(np.int64)
    i1 = i0 + (i0 < n_in - 1)
    l1 = src - i0
    return i0, i1, 1.0 - l1, l1


def upsample(disp, H, W):
    """(N, 1, h, w) -> (N, H, W) fp64: l0y (l0x a + l1x b) + l1y (l0x c + l1x d)"""
    d = disp[:, 0].astype(f64)
    y0, y1, ly0, ly1 = _axis_taps(d.shape[1], H)
    x0, x1, lx0, lx1 = _axis_taps(d.shape[2], W)
    r0, r1 = d[:, y0], d[:, y1]
    top = lx0 * r0[:, :, x0] + lx1 * r0[:, :, x1]
    bot = lx0 * r1[:, :, x0] + lx1 * r1[:, :, x1]
    return ly0[:, None] * top + ly1[:, None] * bot


def upsample_adjoint(g, h, w):
    """the transpose of upsample: (N, H, W) -> (N, h, w)"""
    N, H, W = g.shape
    y0, y1, ly0, ly1 = _axis_taps(h, H)
    x0, x1, lx0, lx1 = _axis_taps(w, W)
    gx = np.zeros((N, H, w))
    for i, l in ((x0, lx0), (x1, lx1)):
        np.add.at(gx, (slice(None), slice(None), i), g * l)
    out = np.zeros((N, h, w))
    for i, l in ((y0, ly0), (y1, ly1)):
        np.add.at(out, (slice(None), i), gx * l[:, None])
    return out


def depth_from_disp(up, min_depth, max_depth):
    """disp_to_depth in fp64: (scaled, depth)"""
    lo, hi = 1.0 / max_depth, 1.0 / min_depth
    scaled = lo + (hi - lo) * up
    return scaled, 1.0 / scaled


def project(D, K, inv_K, T):
    """(N, H, W) depth -> ix, iy (unclipped source coordinates of grid_sample) and d ix / dD, d iy / dD.
    P = K T in fp64 (each element summed over k = 0..3 in order), ray = inv_K[:3, :3] (x, y, 1), a = P[:3, :3] ray,
    q = D a + P[:, 3], u = q0 / (q2 + 1e-7), grid = (u / (W - 1) - 0.5) 2, ix = ((grid + 1) W - 1) / 2."""
    N, H, W = D.shape
    K, Mi, T = K.astype(f64), inv_K.astype(f64), T.astype(f64)
    P = np.zeros((N, 3, 4))
    for i in range(3):
        for j in range(4):
            P[:, i, j] = ((K[:, i, 0] * T[:, 0, j] + K[:, i, 1] * T[:, 1, j]) + K[:, i, 2] * T[:, 2, j]) \
                + K[:, i, 3] * T[:, 3, j]
    ys, xs = np.meshgrid(np.arange(H, dtype=f64), np.arange(W, dtype=f64), indexing="ij")
    e = lambda m: m[:, None, None]                                                       # noqa: E731
    ray = [(e(Mi[:, i, 0]) * xs + e(Mi[:, i, 1]) * ys) + e(Mi[:, i, 2]) for i in range(3)]
    a = [(e(P[:, i, 0]) * ray[0] + e(P[:, i, 1]) * ray[1]) + e(P[:, i, 2]) * ray[2] for i in range(3)]
    b = [e(P[:, i, 3]) for i in range(3)]
    q = [D * a[i] + b[i] for i in range(3)]
    z = q[2] + PROJ_EPS
    u, v = q[0] / z, q[1] / z
    ix = ((((u / (W - 1)) - 0.5) * 2.0 + 1.0) * W - 1.0) / 2.0
    iy = ((((v / (H - 1)) - 0.5) * 2.0 + 1.0) * H - 1.0) / 2.0
    # d u / dD = (a0 (b2 + eps) - a2 b0) / z^2; d ix / du = W / (W - 1)
    bz = b[2] + PROJ_EPS
    du = (a[0] * bz - a[2] * b[0]) / (z * z)
    dv = (a[1] * bz - a[2] * b[1]) / (z * z)
    return ix, iy, du * (W / (W - 1.0)), dv * (H / (H - 1.0))


def sample(img, ix, iy):
    """grid_sample(bilinear, border, align_corners=False) in fp64 from (N, C, H, W) at unclipped ix, iy (N, H, W).
    Returns the sample (N, C, H, W) and its derivatives in ix and iy (0 where the clamp is active or on the border)."""
    N, C, H, W = img.shape
    im = img.astype(f64)
    cx, cy = np.clip(ix, 0.0, W - 1.0), np.clip(iy, 0.0, H - 1.0)
    gate_x = ((ix > 0.0) & (ix < W - 1.0)).astype(f64)
    gate_y = ((iy > 0.0) & (iy < H - 1.0)).astype(f64)
    bad = np.isnan(cx) | np.isnan(cy)
    cx, cy = np.where(bad, 0.0, cx), np.where(bad, 0.0, cy)
    x0, y0 = np.floor(cx).astype(np.int64), np.floor(cy).astype(np.int64)
    x1, y1 = x0 + 1, y0 + 1
    wx1, wy1 = cx - x0, cy - y0
    wx0, wy0 = x1 - cx, y1 - cy
    n = np.arange(N)[:, None, None]

    def tap(yy, xx):
        ok = (xx < W) & (yy < H)
        v = im[n, :, np.minimum(yy, H - 1), np.minimum(xx, W - 1)]       # (N, H, W, C)
        return np.where(ok[..., None], v, 0.0).transpose(0, 3, 1, 2)

    nw, ne, sw, se = tap(y0, x0), tap(y0, x1), tap(y1, x0), tap(y1, x1)
    out = ((nw * (wx0 * wy0)[:, None] + ne * (wx1 * wy0)[:, None]) + sw * (wx0 * wy1)[:, None]) \
        + se * (wx1 * wy1)[:, None]
    out = np.where(bad[:, None], np.nan, out)
    dx = (wy0[:, None] * (ne - nw) + wy1[:, None] * (se - sw)) * gate_x[:, None]
    dy = (wx0[:, None] * (sw - nw) + wx1[:, None] * (se - ne)) * gate_y[:, None]
    return out, dx, dy


def _refl(x):
    return np.pad(x, ((0, 0), (0, 0), (1, 1), (1, 1)), mode="reflect")


def _pool(x):
    """3x3 mean over the reflected window: row sums (dy = -1, 0, 1), then the three rows, then / 9"""
    p = _refl(x)
    H, W = x.shape[2:]
    rows = [(p[:, :, dy:dy + H, 0:W] + p[:, :, dy:dy + H, 1:W + 1]) + p[:, :, dy:dy + H, 2:W + 2] for dy in range(3)]
    return ((rows[0] + rows[1]) + rows[2]) / 9.0


def ssim_parts(x, y):
    """per-pixel SSIM loss (before the clamp gate is applied) and its window coefficients, fp64"""
    mx, my = _pool(x), _pool(y)
    sxx = _pool(x * x) - mx * mx
    syy = _pool(y * y) - my * my
    sxy = _pool(x * y) - mx * my
    A = 2.0 * mx * my + C1
    B = 2.0 * sxy + C2
    Cc = mx * mx + my * my + C1
    Dd = sxx + syy + C2
    n, d = A * B, Cc * Dd
    raw = (1.0 - n / d) / 2.0
    return raw, (mx, my, A, B, Cc, Dd, n, d)


def reproj(pred, target, contract):
    """(N, C, H, W) -> (N, H, W): 0.85 mean_c SSIM + 0.15 mean_c |target - pred|, rounded to fp32 in contract mode"""
    raw, _ = ssim_parts(pred, target)
    s = np.clip(raw, 0.0, 1.0)
    l1 = np.abs(target - pred)
    ssim_m = ((s[:, 0] + s[:, 1]) + s[:, 2]) / 3.0
    l1_m = ((l1[:, 0] + l1[:, 1]) + l1[:, 2]) / 3.0
    return _r32(W_SSIM * ssim_m + W_L1 * l1_m, contract)


def reproj_adjoint(pred, target, wgt):
    """d(sum_q wgt_q reproj_q) / d pred, (N, C, H, W); wgt (N, H, W) is the per-centre weight"""
    raw, (mx, my, A, B, Cc, Dd, n, d) = ssim_parts(pred, target)
    gate = ((raw >= 0.0) & (raw <= 1.0)).astype(f64)                  # clamp passes on [0, 1]; NaN gives 0
    w = (wgt * (W_SSIM / 3.0))[:, None] * gate
    # d ssim_q / d x_j = alpha + beta y_j + gamma x_j for each x_j of q's reflected window
    alpha = -(my * (B - A) / d - n * mx * (Dd - Cc) / (d * d)) / 9.0
    beta = -(A / d) / 9.0
    gamma = (n * Cc / (d * d)) / 9.0
    acc = np.zeros_like(pred, dtype=f64)
    for coef, factor in ((alpha, 1.0), (beta, target), (gamma, pred)):
        s = np.zeros_like(acc)
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                s += _gather_refl(w * coef, dy, dx)
        acc += s * factor
    sgn = np.sign(pred - target)                                      # d |t - p| / dp, sign(0) = 0
    return acc + (wgt * (W_L1 / 3.0))[:, None] * sgn


def _gather_refl(c, dy, dx):
    """sum over centres q with refl(q + (dy, dx)) == j of c[q], for every j: the adjoint of reading a reflected window"""
    N, C, H, W = c.shape
    out = np.zeros_like(c)
    ry = [(q, _reflect(q + dy, H)) for q in range(H)]
    rx = [(q, _reflect(q + dx, W)) for q in range(W)]
    qy = np.array([q for q, _ in ry]); jy = np.array([j for _, j in ry])
    qx = np.array([q for q, _ in rx]); jx = np.array([j for _, j in rx])
    tmp = np.zeros_like(c)
    np.add.at(tmp, (slice(None), slice(None), jy), c[:, :, qy])
    np.add.at(out, (slice(None), slice(None), slice(None), jx), tmp[:, :, :, qx])
    return out


def _reflect(i, n):
    return -i if i < 0 else (2 * (n - 1) - i if i >= n else i)


def smooth(disp, img):
    """get_smooth_loss(disp / (mean + 1e-7), img) in fp64, and its gradient in disp (N, h, w)"""
    d = disp[:, 0].astype(f64)
    im = img.astype(f64)
    N, h, w = d.shape
    mu = d.reshape(N, -1).sum(1) / (h * w)
    den = (mu + 1e-7)[:, None, None]
    nd = d / den
    ex = np.exp(-2.0 * (np.abs(im[:, :, :, :-1] - im[:, :, :, 1:]).sum(1) / 3.0))
    ey = np.exp(-2.0 * (np.abs(im[:, :, :-1, :] - im[:, :, 1:, :]).sum(1) / 3.0))
    gx = nd[:, :, :-1] - nd[:, :, 1:]
    gy = nd[:, :-1, :] - nd[:, 1:, :]
    cx, cy = N * h * (w - 1), N * (h - 1) * w
    with np.errstate(invalid="ignore"):       # one row or one column: the mean over no edges is NaN, as torch's is
        val = (np.abs(gx) * ex).sum() / cx + (np.abs(gy) * ey).sum() / cy
    G = np.zeros_like(d)                                            # d val / d nd
    tx, ty = np.sign(gx) * ex / cx, np.sign(gy) * ey / cy
    G[:, :, :-1] += tx
    G[:, :, 1:] -= tx
    G[:, :-1, :] += ty
    G[:, 1:, :] -= ty
    corr = (G * d).reshape(N, -1).sum(1) / (h * w)
    grad = G / den - (corr / (mu + 1e-7) ** 2)[:, None, None]
    return val, grad


def run(inputs, disps, noise, scales=SCALES, loss_scales=SCALES, min_depth=0.1, max_depth=100.0,
        disparity_smoothness=1e-3, mode="contract", grads=True, grad_terms=None):
    """inputs: "target" color(0, 0) and "source" color("s", 0) (N, 3, H, W), "colors" {s: color(0, s)}, "K", "inv_K",
    "stereo_T" (N, 4, 4), "depth_hint", "depth_hint_mask" (N, 1, H, W); disps {s: (N, 1, H >> s, W >> s)};
    noise {s: (N, 1, H, W) float32 standard normals}.  Returns a dict of the terms ("reproj_loss/s", ...), "warped"
    {s}, "color_depth_hint", "identity_selection" {s}, "depth_hint_pixels" {s} and, with grads, "grad" {s} of "loss",
    or of sum_k grad_terms[k] terms[k] (terms in term_keys(loss_scales) order) when grad_terms is given."""
    c = mode == "contract"
    tgt, src = inputs["target"].astype(f64), inputs["source"].astype(f64)
    N, _, H, W = tgt.shape
    K, iK, T = inputs["K"], inputs["inv_K"], inputs["stereo_T"]
    hint = inputs["depth_hint"][:, 0].astype(f64)
    hmask = inputs["depth_hint_mask"][:, 0].astype(f64)
    out = {"warped": {}, "identity_selection": {}, "depth_hint_pixels": {}, "grad": {}}
    # static maps
    ix, iy, _, _ = project(hint, K, iK, T)
    chint = _r32(sample(src, ix, iy)[0], c)
    out["color_depth_hint"] = chint
    ident = reproj(src, tgt, c)
    hpen = np.float32(HINT_PENALTY) * (np.float32(1.0) - inputs["depth_hint_mask"][:, 0].astype(f32))
    hloss = reproj(chint, tgt, c)
    hloss = (hloss.astype(f32) + hpen).astype(f64) if c else hloss + hpen.astype(f64)
    total = 0.0
    per = {}
    for s in loss_scales:
        up = upsample(disps[s], H, W)
        scaled, D = depth_from_disp(up, min_depth, max_depth)
        ix, iy, dix, diy = project(D, K, iK, T)
        warped, sdx, sdy = sample(src, ix, iy)
        warped = _r32(warped, c)
        out["warped"][s] = warped
        r = reproj(warped, tgt, c)
        nz = (noise[s][:, 0].astype(f32) * NOISE_SCALE).astype(f64)
        ids = (ident.astype(f32) + nz.astype(f32)).astype(f64) if c else ident + nz
        stack = np.stack([r, ids, hloss])
        k = np.where(np.isnan(stack).any(0), np.argmax(np.isnan(stack), 0), np.argmin(np.where(np.isnan(stack), 0, stack), 0))
        rm, hm = (k != 1).astype(f64), (k == 2).astype(f64)
        out["identity_selection"][s] = 1.0 - rm
        out["depth_hint_pixels"][s] = hm
        M, Mh = _count(rm.sum(), c), _count(hm.sum(), c)
        t_rep = _r32(np.asarray((r * rm).sum() / M), c)
        diff = D - hint
        t_hint = _r32(np.asarray((np.log(np.abs(diff) + 1.0) * hmask * hm).sum() / Mh), c)
        sm, sgrad = smooth(disps[s], inputs["colors"][s])
        loss_s = _r32(np.asarray(t_rep + t_hint + disparity_smoothness * sm / 2 ** s), c)
        out["reproj_loss/%d" % s], out["depth_hint_loss/%d" % s], out["loss/%d" % s] = t_rep, t_hint, loss_s
        total = total + loss_s
        per[s] = (D, scaled, dix, diy, sdx, sdy, warped, rm, hm, M, Mh, diff, sgrad)
    out["loss"] = _r32(np.asarray(total / len(scales)), c)
    if not grads:
        return out
    gt = np.zeros(1 + 3 * len(loss_scales)) if grad_terms is None else np.asarray(grad_terms, f32).astype(f64)
    if grad_terms is None:
        gt[0] = 1.0
    for i, s in enumerate(loss_scales):
        gl = gt[0] / len(scales) + gt[3 + 3 * i]
        g_rep, g_hint, g_sm = gl + gt[1 + 3 * i], gl + gt[2 + 3 * i], gl * disparity_smoothness / 2 ** s
        D, scaled, dix, diy, sdx, sdy, warped, rm, hm, M, Mh, diff, sgrad = per[s]
        dx = reproj_adjoint(warped, tgt, rm * (g_rep / M))          # d L / d warped
        dD = (dx * (sdx * dix[:, None] + sdy * diy[:, None])).sum(1)
        dD = dD + (g_hint / Mh) * hmask * hm * np.sign(diff) / (np.abs(diff) + 1.0)
        dup = dD * -((1.0 / min_depth - 1.0 / max_depth) * D * D)
        h, w = disps[s].shape[2:]
        gd = upsample_adjoint(dup, h, w) + g_sm * sgrad
        out["grad"][s] = _r32(gd[:, None], c)
    return out


OPTIONS = dict(min_depth=0.1, max_depth=100.0, disparity_smoothness=1e-3)      # options.py's defaults


def options(case):
    """the case's min_depth, max_depth and disparity_smoothness (options.py's defaults where it sets none)"""
    return {k: case.get(k, v) for k, v in OPTIONS.items()}


def term_keys(loss_scales):
    """the terms in the device's order: "loss", then per loss scale reproj_loss, depth_hint_loss and loss/s"""
    return ["loss"] + [k % s for s in loss_scales for k in ("reproj_loss/%d", "depth_hint_loss/%d", "loss/%d")]


def term_weights(loss_scales):
    """a weight per term for the weighted-term gradients: 1/2 on the total, and (1 + t + 3 s) / 8 on term t of scale s
    with the sign (-1)^(t + s), so that no two terms of a scale or scales of a term share a weight (all exact in fp32)"""
    return (0.5,) + tuple((-1.0) ** (t + s) * (1 + t + 3 * s) / 8.0 for s in loss_scales for t in range(3))


def _case(**kw):
    kw.setdefault("scales", SCALES)
    kw.setdefault("loss_scales", SCALES)
    kw["weights"] = term_weights(kw["loss_scales"])
    return kw


# fixture cases: 2-frame batches at the two KITTI training sizes, a designed special split, a loss_scales subset; a
# different camera per frame (rotated stereo transforms with y and z baselines), non-default options, odd low-resolution
# shapes, one-pixel-thick scale-3 maps (1 row, 1 column: the smoothness has no edge in that direction) and one frame
CASES = {
    "r96x320": _case(seed=1000, N=2, H=96, W=320),
    "r192x640": _case(seed=2000, N=2, H=192, W=640),
    "subset": _case(seed=3000, N=2, H=96, W=320, loss_scales=(0, 2)),
    "special": _case(seed=4000, N=2, H=64, W=96, random=False, special=True),
    "camera": _case(seed=5000, N=3, H=48, W=128, camera=True, fixture=3),
    "options": _case(seed=6000, N=2, H=64, W=192, loss_scales=(1, 3), min_depth=0.5, max_depth=80.0,
                     disparity_smoothness=0.1, fixture=2),
    "odd": _case(seed=7000, N=3, H=72, W=136, camera=True, fixture=3),
    "thin_row": _case(seed=8000, N=2, H=8, W=64, fixture=2),
    "thin_col": _case(seed=9000, N=2, H=64, W=8, fixture=2),
    "single": _case(seed=10000, N=1, H=64, W=192, fixture=2),
}
# the fixture's files under tests/golden, each well under 1 MiB: the first four cases as they were first pinned, their
# weighted-term gradients (and weights), the cases added with those gradients (options and shapes, then cameras)
FIXTURES = ("kitti_hints_loss.npz", "kitti_hints_loss_terms.npz", "kitti_hints_loss_shapes.npz",
            "kitti_hints_loss_cameras.npz")
FIRST_CASES = ("r96x320", "r192x640", "subset", "special")


def fixture_file(key):
    """which of FIXTURES holds fixture key `key` ("<case>/...")"""
    case, _, rest = key.partition("/")
    if case not in FIRST_CASES:
        return FIXTURES[CASES[case]["fixture"]]
    return FIXTURES[1] if rest == "weights" or rest.startswith("f64/wgrad/") else FIXTURES[0]


def load_fixture(directory):
    """every key of the fixture's files in `directory` as one dict; "cases" lists each file's cases in FIXTURES order"""
    out, cases = {}, []
    for name in FIXTURES:
        with np.load(os.path.join(directory, name)) as f:
            for k in f.files:
                if k == "cases":
                    cases += [str(c) for c in f[k]]
                else:
                    out[k] = f[k]
    out["cases"] = np.array(cases)
    return out


def cameras(N, H, W):
    """per-frame intrinsics as crops and rescales of KITTI's give them (focal lengths and principal points differ per
    frame), their inverses, and stereo transforms with a rotation of 3-7 degrees about each axis and a translation with
    x, y and z components, the signs alternating per frame: warps leave the image on all four sides, every z stays > 0"""
    K = np.zeros((N, 4, 4), np.float32)
    T = np.zeros((N, 4, 4), np.float32)
    for n in range(N):
        sg, grow = (1.0 if n % 2 == 0 else -1.0), 1.0 + 0.25 * n
        fx, fy = 0.58 * W * (1.0 + 0.2 * n), 1.92 * H * (1.0 + 0.1 * n)
        cx, cy = W * (0.5 + 0.04 * sg * (n + 1)), H * (0.5 - 0.06 * sg * (n + 1))
        K[n] = [[fx, 0, cx, 0], [0, fy, cy, 0], [0, 0, 1, 0], [0, 0, 0, 1]]
        ax, ay, az = np.radians([3.0 * sg * grow, -2.5 * sg * grow, 4.0 * sg * grow])
        rx = np.array([[1, 0, 0], [0, np.cos(ax), -np.sin(ax)], [0, np.sin(ax), np.cos(ax)]])
        ry = np.array([[np.cos(ay), 0, np.sin(ay)], [0, 1, 0], [-np.sin(ay), 0, np.cos(ay)]])
        rz = np.array([[np.cos(az), -np.sin(az), 0], [np.sin(az), np.cos(az), 0], [0, 0, 1]])
        T[n, :3, :3] = rz @ ry @ rx
        T[n, :3, 3] = [0.1 * sg, 0.04 * sg * grow, -0.02 * sg * grow]
        T[n, 3, 3] = 1.0
    return K, np.linalg.pinv(K).astype(np.float32), T


def intrinsics(N, H, W):
    """KITTI's normalised intrinsics (kitti_dataset.py) at (H, W), their inverse, and the stereo transform"""
    K = np.array([[0.58 * W, 0, 0.5 * W, 0], [0, 1.92 * H, 0.5 * H, 0], [0, 0, 1, 0], [0, 0, 0, 1]], np.float32)
    inv_K = np.linalg.pinv(K).astype(np.float32)
    T = np.eye(4, dtype=np.float32)
    T[0, 3] = 0.1
    return np.repeat(K[None], N, 0), np.repeat(inv_K[None], N, 0), np.repeat(T[None], N, 0)


def make_inputs(case, seed):
    """(inputs, disps) of a case, float32, from its seed"""
    rng = np.random.default_rng(seed)
    N, H, W = case["N"], case["H"], case["W"]
    r = lambda *s: rng.random(s, dtype=np.float32)                                     # noqa: E731
    K, inv_K, T = (cameras if case.get("camera") else intrinsics)(N, H, W)
    inp = {"target": r(N, 3, H, W), "K": K, "inv_K": inv_K, "stereo_T": T,
           "depth_hint": (1.0 + 40.0 * r(N, 1, H, W)).astype(np.float32),
           "depth_hint_mask": (r(N, 1, H, W) < 0.8).astype(np.float32)}
    # the source: the target shifted by about ten pixels plus noise, so that warps, hints and the identity compete
    inp["source"] = (0.7 * np.roll(inp["target"], -10, axis=3) + 0.3 * r(N, 3, H, W)).astype(np.float32)
    inp["colors"] = {s: r(N, 3, H >> s, W >> s) for s in case["scales"] if s}
    inp["colors"][0] = inp["target"]                                   # ("color", 0, 0) is the target
    disps = {s: (0.02 + 0.08 * r(N, 1, H >> s, W >> s)).astype(np.float32) for s in case["scales"]}
    if case.get("special"):
        inp["depth_hint_mask"][0] = 0.0                                  # frame 0: no hint at all
        inp["depth_hint_mask"][1] = 1.0                                  # frame 1: a hint everywhere
        d0 = disps[0]
        d0[0, 0, :8, :] = 0.0                                            # depth 100: barely moves
        d0[0, 0, 8:16, :] = 1.0                                          # depth 0.1: far off the image's left side
        d0[1, 0, :8, :] = 1.0
        inp["stereo_T"][1, 0, 3] = -0.1                                  # frame 1 moves the other way: off the right
        # exact ties between r and the hint loss: the hint equals every scale's depth at these pixels, so the hint warp
        # and the scale warps read the same colours
        disps[1][1, 0, 16:20, :] = 0.05
        disps[2][1, 0, 8:10, :] = 0.05
        disps[3][1, 0, 4:5, :] = 0.05
        disps[0][1, 0, 32:40, :] = 0.05
        inp["depth_hint"][1, 0, 33:39, 2:-2] = np.float32(1.0 / (0.01 + (10.0 - 0.01) * 0.05))
    return inp, disps


def draw_noise(seed, inputs, loss_scales):
    """the reference's tie-breaking noise: torch.randn((N, 1, H, W)) per loss scale, in order, after manual_seed(seed)"""
    import torch
    N, _, H, W = inputs["target"].shape
    torch.manual_seed(seed)
    return {s: torch.randn((N, 1, H, W)).numpy() for s in loss_scales}


def decision_margin(inputs, disps, noise, case):
    """the smallest relative distance, in fp64, of any argmin or grid-sample floor from its decision (exact ties
    excepted)"""
    opt = options(case)
    out = run(inputs, disps, noise, case["scales"], case["loss_scales"], mode="fp64", grads=False, **opt)
    tgt, src = inputs["target"].astype(f64), inputs["source"].astype(f64)
    N, _, H, W = tgt.shape
    worst = np.inf
    hint = inputs["depth_hint"][:, 0].astype(f64)
    ds = [hint] + [depth_from_disp(upsample(disps[s], H, W), opt["min_depth"], opt["max_depth"])[1]
                   for s in case["loss_scales"]]
    for D in ds:
        ix, iy, _, _ = project(D, inputs["K"], inputs["inv_K"], inputs["stereo_T"])
        for v, n in ((ix, W), (iy, H)):
            inside = (v > 0) & (v < n - 1)
            frac = np.abs(v - np.round(v))[inside] / np.maximum(np.abs(v[inside]), 1.0)
            if frac.size:
                worst = min(worst, frac.min())
    ident = reproj(src, tgt, False)
    hl = reproj(out["color_depth_hint"], tgt, False) + 1000.0 * (1.0 - inputs["depth_hint_mask"][:, 0])
    for s in case["loss_scales"]:
        r = reproj(out["warped"][s], tgt, False)
        ids = ident + (noise[s][:, 0] * NOISE_SCALE).astype(f64)
        st = np.sort(np.stack([r, ids, hl]), 0)
        # an exact tie does not count: r and the hint loss of a pixel whose scale and hint warps both leave the image
        # past the same corner read the same clamped colours, and every precision decides that tie alike (first minimum)
        gap = st[1] - st[0]
        gap = gap[gap != 0]
        if gap.size:
            worst = min(worst, (gap / np.maximum(np.abs(st[0][st[1] != st[0]]), 1e-30)).min())
    return worst
