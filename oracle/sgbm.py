"""numpy restatement of OpenCV's StereoSGBM (MODE_SGBM), bit for bit: ``compute(left, right)`` on uint8 (H, W, 3) images.

Every stage is integer arithmetic, in the order OpenCV applies it:
  * prefilter, per channel: the x-Sobel (2 (r[x+1] - r[x-1]) + the same on the rows above and below, the image's edge
    row standing in for the missing one) clipped to [-cap, cap] and offset by cap, cap = max(preFilterCap, 15) | 1;
    columns 0 and W - 1 of every plane, the raw ones too, hold cap;
  * pixel cost for d in [0, D) at columns x in [D, W) of the left image: Birchfield-Tomasi's min of the two
    half-pixel-interval distances between left column x and right column x - d, summed over the three Sobel planes
    (shift 0) and the three raw planes (each >> 2);
  * block sum over half-width s = blockSize // 2 (blockSize 2 and 3 are one matcher): columns clamped to [D, W - 1],
    rows to [0, H - 1];
  * five aggregation paths (left-to-right, top-left, top, top-right, right-to-left), each
    L = C + min(L'[d], L'[d - 1] + P1, L'[d + 1] + P1, min L' + P2) - min L', starting from L = C; S their sum,
    saturated to int16 at two points (the four forward paths, then the fifth);
  * the winner: the first minimum of S; it is refused if some d with |d - best| > 1 has S (100 - ratio) < min S 100;
  * sub-pixel: 16 d + ((S[d-1] - S[d+1]) 16 + den) / (2 den), den = max(S[d-1] + S[d+1] - 2 S[d], 1), C's truncating
    division, for 0 < d < D - 1;
  * the right view's winner per column: the unique left pixel with the least min S, ties to the larger x (OpenCV walks
    x downwards and replaces on a strictly smaller cost);
  * the left-right check: a pixel is refused when both floor(d) and ceil(d) land on a right winner farther than
    disp12MaxDiff (0 means 1) away;
  * a 3x3 median of the int16 map (cv::medianBlur, edges replicated), invalid pixels included;
  * filterSpeckles: 4-connected components of valid pixels whose neighbours differ by at most speckleRange 16; a
    component of at most speckleWindowSize pixels becomes invalid.
Invalid pixels hold (minDisparity - 1) 16; minDisparity is 0 here, as in the depth-hints matchers.
"""
import numpy as np

MAX_COST = 32767
I32 = np.int32

# the depth-hints matchers' parameters (KITTI/precompute_depth_hints.py, generate_stereo_matchers)
HINT_PARAMS = dict(preFilterCap=63, P1=36, P2=288, uniquenessRatio=10, speckleWindowSize=100, speckleRange=16,
                   disp12MaxDiff=0)
NUM_DISPARITIES = (64, 96, 128, 160)
BLOCK_SIZES = (1, 2, 3)
MATCHERS = tuple((nd, bs) for bs in BLOCK_SIZES for nd in NUM_DISPARITIES)   # the reference's order


def min_width(num_disparities, block_size):
    """the least width OpenCV accepts: width - numDisparities > blockSize // 2"""
    return num_disparities + block_size // 2 + 1


def prefilter(img, cap):
    """(H, W, 3) uint8 -> (6, H, W) int32: the clipped x-Sobel of each channel, then the raw channels"""
    ftzero = max(cap, 15) | 1
    im = img.astype(I32)
    H, W, _ = im.shape
    up = np.concatenate([im[:1], im[:-1]], 0)
    dn = np.concatenate([im[1:], im[-1:]], 0)
    out = np.full((6, H, W), ftzero, I32)
    for c in range(3):
        g = (im[:, 2:, c] - im[:, :-2, c]) * 2 + up[:, 2:, c] - up[:, :-2, c] + dn[:, 2:, c] - dn[:, :-2, c]
        out[c, :, 1:-1] = np.clip(g, -ftzero, ftzero) + ftzero
        out[3 + c, :, 1:-1] = im[:, 1:-1, c]
    return out


def _half_minmax(p):
    """per column: min and max of the value and its two half-pixel neighbours (x +- 1/2, floor division)"""
    left = np.concatenate([p[..., :1] * 2, p[..., :-1] + p[..., 1:]], -1) // 2
    right = np.concatenate([p[..., :-1] + p[..., 1:], p[..., -1:] * 2], -1) // 2
    return np.minimum(np.minimum(left, right), p), np.maximum(np.maximum(left, right), p)


def pixel_cost(left, right, D, cap):
    """(H, W - D, D) int32: the Birchfield-Tomasi cost of left column D + i against right column D + i - d"""
    a, b = prefilter(left, cap), prefilter(right, cap)
    a0, a1 = _half_minmax(a)
    b0, b1 = _half_minmax(b)
    _, H, W = a.shape
    xs = np.arange(D, W)[:, None] - np.arange(D)[None, :]            # right column (W - D, D)
    cost = np.zeros((H, W - D, D), I32)
    for c in range(6):
        u, u0, u1 = a[c][:, D:, None], a0[c][:, D:, None], a1[c][:, D:, None]
        v, v0, v1 = b[c][:, xs], b0[c][:, xs], b1[c][:, xs]
        c0 = np.maximum(np.maximum(0, u - v1), v0 - u)
        c1 = np.maximum(np.maximum(0, v - u1), u0 - v)
        cost += np.minimum(c0, c1) >> (0 if c < 3 else 2)
    return cost


def block_cost(pix, half):
    """the block sum of the pixel cost over (2 half + 1)^2, OpenCV's clamps (see the module docstring)"""
    H, W1, _ = pix.shape
    if half == 0:
        return pix.copy()
    cols = np.clip(np.arange(W1)[:, None] + np.arange(-half, half + 1)[None, :], 0, W1 - 1)
    hs = pix[:, cols].sum(2)                                          # (H, W1, D)
    rows = np.clip(np.arange(H)[:, None] + np.arange(-half, half + 1)[None, :], 0, H - 1)
    return hs[rows].sum(1)


def _wrap16(v):
    return ((v + 32768) & 0xFFFF) - 32768


def _sat16(v):
    return np.clip(v, -32768, 32767)


def _step(C, Lp, P1, P2):
    """one path step over the last axis (disparity): C + min(Lp, Lp[d-1] + P1, Lp[d+1] + P1, min Lp + P2) - min Lp.
    A previous pixel outside the image is Lp = 0, which gives L = C."""
    m = Lp.min(-1, keepdims=True)
    big = np.full(Lp.shape[:-1] + (1,), MAX_COST, I32)
    lo = np.concatenate([big, Lp[..., :-1]], -1) + P1
    hi = np.concatenate([Lp[..., 1:], big], -1) + P1
    return _wrap16(C + np.minimum(np.minimum(Lp, lo), np.minimum(hi, m + P2)) - m)


def aggregate(C, P1, P2):
    """(H, W1, D) block cost -> S (int32 holding int16 values): the five paths' sum, saturated to int16 after the four
    forward paths and again after the right-to-left one"""
    H, W1, D = C.shape
    zero_col = np.zeros((H, D), I32)
    fwd = np.zeros((H, W1, D), I32)
    L = zero_col
    for x in range(W1):                                               # left to right
        L = _step(C[:, x], L, P1, P2)
        fwd[:, x] += L
    zero_row = np.zeros((1, D), I32)
    prev = [np.zeros((W1, D), I32)] * 3
    for y in range(H):                                                # from x - 1, x, x + 1 of the row above
        srcs = (np.concatenate([zero_row, prev[0][:-1]]), prev[1], np.concatenate([prev[2][1:], zero_row]))
        prev = [_step(C[y], s, P1, P2) for s in srcs]
        fwd[y] += prev[0] + prev[1] + prev[2]
    S = _sat16(fwd)
    L = zero_col
    for x in range(W1 - 1, -1, -1):                                   # right to left
        L = _step(C[:, x], L, P1, P2)
        S[:, x] = _sat16(S[:, x] + L)
    return S


def _cdiv(a, b):
    """C's integer division (truncates toward zero), b > 0"""
    q = np.abs(a) // b
    return np.where(a < 0, -q, q)


def select(S, W, D, uniqueness, disp12):
    """(H, W1, D) S -> (H, W) int32 disparity x16 after the uniqueness check, the sub-pixel fit and the left-right check"""
    H, W1, _ = S.shape
    inv = -16
    best = S.argmin(-1)                                               # the first minimum
    minS = np.take_along_axis(S, best[..., None], -1)[..., 0]
    d = np.arange(D)
    far = np.abs(best[..., None] - d) > 1
    unique = ~((S * (100 - uniqueness) < minS[..., None] * 100) & far).any(-1)
    sm = np.take_along_axis(S, np.clip(best - 1, 0, D - 1)[..., None], -1)[..., 0]
    sp = np.take_along_axis(S, np.clip(best + 1, 0, D - 1)[..., None], -1)[..., 0]
    den = np.maximum(sm + sp - 2 * minS, 1)
    inner = (best > 0) & (best < D - 1)
    sub = np.where(inner, best * 16 + _cdiv((sm - sp) * 16 + den, den * 2), best * 16)
    disp = np.full((H, W), inv, I32)
    disp[:, D:] = np.where(unique, sub, inv)
    # the right view's winners: OpenCV walks x from W1 - 1 down and replaces on a strictly smaller cost
    disp2 = np.full((H, W), inv, I32)
    cost2 = np.full((H, W), MAX_COST, I32)
    for x in range(W1 - 1, -1, -1):
        x2 = x + D - best[:, x]
        rows = np.nonzero(unique[:, x] & (cost2[np.arange(H), x2] > minS[:, x]))[0]
        cost2[rows, x2[rows]] = minS[rows, x]
        disp2[rows, x2[rows]] = best[rows, x]
    maxdiff = disp12 if disp12 > 0 else 1
    out = disp.copy()
    xs = np.arange(W)[None, :].repeat(H, 0)
    ys = np.arange(H)[:, None].repeat(W, 1)

    def bad(dd):
        xx = xs - dd
        ok = (xx >= 0) & (xx < W)
        v = disp2[ys, np.clip(xx, 0, W - 1)]
        return ok & (v >= 0) & (np.abs(v - dd) > maxdiff)

    lo, hi = disp >> 4, (disp + 15) >> 4
    out[(disp != inv) & bad(lo) & bad(hi)] = inv
    return out


def median3(disp):
    """cv::medianBlur(disp, 3) on int16: the median of each 3x3 window, edges replicated"""
    p = np.pad(disp, 1, mode="edge")
    H, W = disp.shape
    win = np.stack([p[dy:dy + H, dx:dx + W] for dy in range(3) for dx in range(3)])
    return np.sort(win, 0)[4]


def filter_speckles(disp, new_val, max_size, max_diff):
    """cv::filterSpeckles: invalidate 4-connected components (neighbours within max_diff) of at most max_size pixels"""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    H, W = disp.shape
    ok = disp != new_val
    idx = np.arange(H * W).reshape(H, W)
    e_h = ok[:, :-1] & ok[:, 1:] & (np.abs(disp[:, :-1] - disp[:, 1:]) <= max_diff)
    e_v = ok[:-1] & ok[1:] & (np.abs(disp[:-1] - disp[1:]) <= max_diff)
    a = np.concatenate([idx[:, :-1][e_h], idx[:-1][e_v]])
    b = np.concatenate([idx[:, 1:][e_h], idx[1:][e_v]])
    g = coo_matrix((np.ones(a.size, np.int8), (a, b)), shape=(H * W, H * W))
    _, lab = connected_components(g, directed=False)
    size = np.bincount(lab, minlength=lab.max() + 1)
    out = disp.copy()
    out[ok & (size[lab].reshape(H, W) <= max_size)] = new_val
    return out


def compute(left, right, numDisparities, blockSize, preFilterCap=63, P1=36, P2=288, uniquenessRatio=10,
            speckleWindowSize=100, speckleRange=16, disp12MaxDiff=0):
    """cv2.StereoSGBM_create(minDisparity=0, ...).compute(left, right) on uint8 (H, W, 3): (H, W) int16"""
    H, W, _ = left.shape
    D, half = numDisparities, blockSize // 2
    if D % 16 or D <= 0 or W - D <= half:
        raise ValueError("width %d too small for numDisparities %d and blockSize %d" % (W, D, blockSize))
    P1 = P1 if P1 > 0 else 2
    P2 = max(P2 if P2 > 0 else 5, P1 + 1)
    C = block_cost(pixel_cost(left, right, D, preFilterCap), half)
    S = aggregate(C, P1, P2)
    disp = median3(select(S, W, D, uniquenessRatio if uniquenessRatio >= 0 else 10, disp12MaxDiff))
    if speckleWindowSize > 0:
        disp = filter_speckles(disp, -16, speckleWindowSize, 16 * speckleRange)
    return disp.astype(np.int16)


def compute_side(left, right, numDisparities, blockSize, reverse, **kw):
    """the depth-hints script's matcher call: with reverse (the base view is the right one) both views are mirrored
    around the matcher and the result is mirrored back"""
    if reverse:
        return compute(left[:, ::-1], right[:, ::-1], numDisparities, blockSize, **kw)[:, ::-1]
    return compute(left, right, numDisparities, blockSize, **kw)
