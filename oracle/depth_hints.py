"""numpy restatement of KITTI's depth-hints fusion (KITTI/precompute_depth_hints.py: compute_depths and run), the
contract of include/wmd_hints.h's wmd_depth_hints_f32.

Per view: the twelve matchers' int16 maps (oracle.sgbm, the script's order), ``disp = map / 16``, ``depth = K00 0.1 /
(disp + 1e-7) (disp > 0)`` at the script's float32 rounding points (-0.0 where the quotient is negative), the lookup
view (uint8 / 255 in float32) warped by each depth and scored against the base view with oracle.kitti_loss's
``project``, ``sample`` and ``reproj`` (the loss and the fusion share the device code too), then torch.argmin over the
twelve (the first NaN, else the first minimum) and the winning depth.

Two modes, as oracle.kitti_loss: ``contract`` rounds the warped colours and each reprojection error to float32, as the
device does; ``fp64`` rounds nothing, to be held to the script's own float64 run.
"""
import numpy as np

from oracle import kitti_loss as okl
from oracle import sgbm

f32, f64 = np.float32, np.float64
BASELINE = 0.1


def cameras(height, width, right):
    """the script's K (float32, row 0 scaled by W and row 1 by H in float32), inv_K = pinv(K) and the stereo transform
    T[0, 3] = +-0.1 (right views +), each (N, 4, 4) float32"""
    K = np.array([[0.58, 0, 0.5, 0], [0, 1.92, 0.5, 0], [0, 0, 1, 0], [0, 0, 0, 1]], dtype=f32)
    K[0] *= width
    K[1] *= height
    inv_K = np.linalg.pinv(K)
    right = np.asarray(right, bool).reshape(-1)
    T = np.repeat(np.eye(4, dtype=f32)[None], right.size, 0)
    T[:, 0, 3] = np.where(right, f32(BASELINE), f32(-BASELINE))
    n = right.size
    return np.repeat(K[None], n, 0), np.repeat(inv_K[None], n, 0), T


def depths(maps, k00):
    """(..., H, W) int16 maps -> float32 depths: fp32(fp32(k00 0.1) / fp32(disp + 1e-7)) * (disp > 0)"""
    disp = (maps / 16).astype(f32)
    num = f32(k00) * f32(BASELINE)
    return (num / (disp + f32(1e-7))) * (disp > 0).astype(f32)


def planes(views):
    """(N, H, W, 3) uint8 -> (N, 3, H, W) float32 u / 255"""
    return views.astype(f32).transpose(0, 3, 1, 2) / f32(255)


def argmin_first(stack):
    """torch.argmin over axis 0: the first NaN, else the first minimum"""
    nan = np.isnan(stack)
    return np.where(nan.any(0), np.argmax(nan, 0), np.argmin(np.where(nan, np.inf, stack), 0))


def fuse(base, lookup, maps, right, mode="contract"):
    """base, lookup (N, H, W, 3) uint8; maps (12, N, H, W) int16; right (N) bools -> (depth (N, 1, H, W) float32,
    index (N, 1, H, W) int64, errors (12, N, H, W) fp64)"""
    c = mode == "contract"
    N, H, W, _ = base.shape
    K, inv_K, T = cameras(H, W, right)
    tgt, src = planes(base).astype(f64), planes(lookup).astype(f64)
    D = np.stack([depths(maps[:, n], K[n, 0, 0]) for n in range(N)], 1)      # (12, N, H, W) float32
    errs = []
    for m in range(maps.shape[0]):
        ix, iy, _, _ = okl.project(D[m].astype(f64), K, inv_K, T)
        warped = okl._r32(okl.sample(src, ix, iy)[0], c)
        errs.append(okl.reproj(warped, tgt, c))
    errs = np.stack(errs)
    k = argmin_first(errs)
    best = np.take_along_axis(D, k[None], 0)[0]
    return best[:, None], k[:, None], errs


TIE_REL = 1e-12


def check_fp64(errs, depth, index, ref_index, ref_depth):
    """errs, depth (12, H, W): the fp64 mode's errors and the matchers' depths; index (H, W) its argmin; ref_index,
    ref_depth the float64 reference's.  The reference's depth must be its own matcher's depth, bit for bit, and that
    matcher's error must lie within TIE_REL (relative) of the oracle's least error.  Where several matchers' errors
    are that close (their warps read the same or nearly the same colours), the reference's own float64 rounding (its
    batched matmul and grid arithmetic) picks among them.  Returns the number of pixels whose index differs, or None
    on a mismatch."""
    pick = np.take_along_axis(errs, ref_index[None], 0)[0]
    best = np.take_along_axis(errs, index[None], 0)[0]
    close = (np.abs(pick - best) <= TIE_REL * np.abs(best)) | (np.isnan(pick) & np.isnan(best))
    own = np.take_along_axis(depth, ref_index[None], 0)[0]
    if not (close.all() and (own.astype(f32).view(np.uint32) == ref_depth.astype(f32).view(np.uint32)).all()):
        return None
    return int((index != ref_index).sum())


def matcher_maps(base, lookup, right, **kw):
    """oracle.sgbm's twelve maps (12, N, H, W) int16 in the script's order, right views mirrored around the matcher"""
    out = []
    for nd, bs in sgbm.MATCHERS:
        out.append(np.stack([sgbm.compute_side(base[n], lookup[n], nd, bs, bool(r), **kw)
                             for n, r in enumerate(np.asarray(right, bool).reshape(-1))]))
    return np.stack(out)


def _texture(rng, h, w, cell):
    """blocky random colour texture, each block averaged with its neighbours (uint8-range int32)"""
    t = rng.integers(0, 256, (h // cell + 2, w // cell + 2, 3))
    t = np.repeat(np.repeat(t, cell, 0), cell, 1)[:h, :w]
    return (t + np.roll(t, 1, 0) + np.roll(t, 1, 1) + np.roll(t, (1, 1), (0, 1))) // 4


def make_pair(seed, H, W):
    """a synthetic rectified pair (left, right), (H, W, 3) uint8, numpy only: a textured background and three textured
    layers at seeded disparities up to 150 (occlusions where a nearer layer covers a farther one), a textureless patch,
    saturated 0 and 255 patches, a repetitive stripe patch, and independent noise on the right view"""
    rng = np.random.default_rng(seed)
    db = int(rng.integers(3, 24))
    bg = _texture(rng, H, W + db, int(rng.integers(2, 5)))
    left, right = bg[:, :W].copy(), bg[:, db:db + W].copy()
    for d in sorted(int(v) for v in rng.integers(db + 4, min(150, W - 8), 3)):      # far to near
        w = int(rng.integers(W // 8, W // 3))
        x0 = int(rng.integers(d, max(d + 1, W - w)))
        w = min(w, W - x0)
        y0, y1 = sorted(int(v) for v in rng.integers(0, H + 1, 2))
        if y1 - y0 < 2:
            y0, y1 = 0, H
        tex = _texture(rng, H, W + d, int(rng.integers(1, 4)))
        left[y0:y1, x0:x0 + w] = tex[y0:y1, x0:x0 + w]
        xs = np.arange(max(x0 - d, 0), min(x0 + w - d, W))
        right[y0:y1, xs] = tex[y0:y1, xs + d]
    # a textureless, a black, a white and a striped patch, each at the background's disparity in both views
    for k, fill in enumerate((128, 0, 255, None)):
        ph, pw = max(H // 6, 1), max(W // 10, 2)
        y, x = int(rng.integers(0, H - ph + 1)), int(rng.integers(db + 1, W - pw + 1))
        if fill is None:
            stripe = ((np.arange(W + db) // 4) % 2 * 200 + 20)[None, :, None]
            left[y:y + ph, x:x + pw] = stripe[:, x:x + pw]
            right[y:y + ph, x - db:x - db + pw] = stripe[:, x:x + pw]
        else:
            left[y:y + ph, x:x + pw] = fill
            right[y:y + ph, x - db:x - db + pw] = fill
    right = right + rng.integers(-6, 7, right.shape)
    return np.clip(left, 0, 255).astype(np.uint8), np.clip(right, 0, 255).astype(np.uint8)


def sample_pair(image, H, W):
    """a pair from one (h, w, 3) uint8 photograph resized to (W, H) (LANCZOS): the left view is the photo, the right
    view reads it at x + d with d rising by rows from 8 to 120 in three bands, as a scene of three depths would"""
    from PIL import Image
    left = np.asarray(Image.fromarray(image).resize((W, H), Image.LANCZOS), dtype=np.uint8)
    d = np.where(np.arange(H) < H // 3, 8, np.where(np.arange(H) < 2 * H // 3, 40, 120))
    xs = np.minimum(np.arange(W)[None, :] + d[:, None], W - 1)
    right = left[np.arange(H)[:, None], xs]
    return left, np.ascontiguousarray(right)


# fixture cases: (seed, H, W); the small ones are stored whole, the full-size ones as digests
SMALL = {"a": (101, 64, 256), "b": (202, 64, 256), "c": (303, 96, 320)}
FULL = {"full0": (404, 320, 1024), "full1": (505, 320, 1024)}
CV2_VERSION = "4.13.0"


def views(left, right, side):
    """(base, lookup, reverse) of a pair for the script's side "l" or "r" """
    return (left, right, False) if side == "l" else (right, left, True)
