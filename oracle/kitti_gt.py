"""numpy restatement of KITTI's ground-truth export (KITTI/kitti_utils.py:45-104, generate_depth_map), the contract of
include/wmd_gt.h's wmd_velo_depth_f64, and the synthetic data its fixtures are made of.

Per frame, with P = P_rect_0{cam} . R_cam2rect . velo2cam (3x4 fp64) and (H, W) from S_rect_02:
  * points with x >= 0 (file order; NaN x dropped, -0.0 kept) are projected as np.dot(P, velo.T) does it:
    q_r = fma(P[r][3], 1, fma(P[r][2], z, fma(P[r][1], y, P[r][0] x))) in fp64 (the reflectance is replaced by 1);
  * u' = rint(q0 / q2) - 1, v' = rint(q1 / q2) - 1 (half to even); kept if 0 <= u' < W and 0 <= v' < H;
  * the point's depth is x if vel_depth, else q2;
  * each pixel takes the depth of the LAST kept point on it;
  * duplicate groups g = v' (W - 1) + u' - 1 (sub2ind's off-by-one: (y, W-1) and (y+1, 0) share a group): where a
    group has more than one point, the pixel of its FIRST point takes the group minimum (of equal zeros, the later
    point's, as numpy's min returns for such groups);
  * depth < 0 becomes 0 (-0.0 stays).
"""
import os

import numpy as np

f32, f64 = np.float32, np.float64

# ----------------------------------------------------------------------------------------------------- exact fp64 fma
_SPLIT = f64(134217729.0)                                    # 2^27 + 1, Veltkamp's splitter for 53-bit doubles


def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _two_prod(a, b):
    p = a * b
    ca, cb = _SPLIT * a, _SPLIT * b
    ah, bh = ca - (ca - a), cb - (cb - b)
    al, bl = a - ah, b - bh
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _add_round_odd(a, b):
    """a + b rounded to odd: the rounded sum, moved one ulp toward the exact sum when that is inexact and even"""
    s, e = _two_sum(a, b)
    even = (s.view(np.int64) & 1) == 0
    return np.where((e != 0) & even, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)


def fma(a, b, c):
    """a * b + c rounded once (Boldo and Melquiond's emulation through rounding to odd), elementwise in fp64; exact
    for finite operands whose products neither overflow nor underflow; non-finite operands take the plain a * b + c,
    which has the same class (NaN or the same infinity)"""
    a, b, c = (np.asarray(v, f64) for v in (a, b, c))
    a, b, c = np.broadcast_arrays(a, b, c)
    with np.errstate(all="ignore"):
        uh, ul = _two_prod(a, b)
        th, tl = _two_sum(c, ul)
        vh, vl = _two_sum(uh, th)
        r = vh + _add_round_odd(vl, tl)
        return np.where(np.isfinite(a) & np.isfinite(b) & np.isfinite(c), r, a * b + c)


# ----------------------------------------------------------------------------------------------------- the contract
def project(points, P):
    """(M, 4) float32 points -> (M, 3) fp64 q, np.dot(P, velo.T).T with the reflectance replaced by 1"""
    x, y, z = (points[:, k].astype(f64) for k in range(3))
    P = np.asarray(P, f64)
    with np.errstate(all="ignore"):
        return np.stack([fma(P[r, 3], 1.0, fma(P[r, 2], z, fma(P[r, 1], y, P[r, 0] * x))) for r in range(3)], 1)


def kept_points(points, P, H, W, vel_depth):
    """indices (into points), u', v' (int64) and depths (fp64) of the kept points, in file order"""
    points = np.asarray(points, f32).reshape(-1, 4)
    q = project(points, P)
    x = points[:, 0].astype(f64)
    with np.errstate(all="ignore"):
        u = np.rint(q[:, 0] / q[:, 2]) - 1
        v = np.rint(q[:, 1] / q[:, 2]) - 1
    keep = (x >= 0) & (u >= 0) & (v >= 0) & (u < W) & (v < H)
    idx = np.nonzero(keep)[0]
    d = (x if vel_depth else q[:, 2])[idx]
    return idx, u[idx].astype(np.int64), v[idx].astype(np.int64), d


def depth_map(points, P, H, W, vel_depth=False):
    """generate_depth_map's (H, W) fp64 map for one scan"""
    _, u, v, d = kept_points(points, P, H, W, vel_depth)
    depth = np.zeros(H * W, f64)
    if d.size == 0:
        return depth.reshape(H, W)
    k = np.arange(d.size)
    pix = v * W + u
    last = np.full(H * W, -1, np.int64)
    np.maximum.at(last, pix, k)
    hit = last >= 0
    depth[hit] = d[last[hit]]
    g = v * (W - 1) + u - 1
    # per group: its first point, its size, and its least depth (zeros compare equal; of those the later point)
    groups, first, count = np.unique(g, return_index=True, return_counts=True)
    order = np.lexsort((-k, d + 0.0, g))                  # by group, then value (-0 == +0), then later point first
    gs = g[order]
    head = order[np.r_[True, gs[1:] != gs[:-1]]]          # the least point of each group, in ascending group order
    dup = count > 1
    depth[pix[first[dup]]] = d[head[dup]]
    depth[depth < 0] = 0
    return depth.reshape(H, W)


# ----------------------------------------------------------------------------------------------------- calibration
def read_calib_text(text):
    """kitti_utils.read_calib_file on a string"""
    float_chars = set("0123456789.e+- ")
    data = {}
    for line in text.splitlines(True):
        key, value = line.split(":", 1)
        value = value.strip()
        data[key] = value
        if float_chars.issuperset(value):
            try:
                data[key] = np.array(list(map(float, value.split(" "))))
            except ValueError:
                pass
    return data


def velo_to_image(cam2cam, velo2cam, cam):
    """(P (3, 4) fp64, (H, W)) from the two parsed calibration files, as generate_depth_map forms them"""
    Rt = np.hstack((velo2cam["R"].reshape(3, 3), velo2cam["T"][..., np.newaxis]))
    Rt = np.vstack((Rt, np.array([0, 0, 0, 1.0])))
    R_cam2rect = np.eye(4)
    R_cam2rect[:3, :3] = cam2cam["R_rect_00"].reshape(3, 3)
    P_rect = cam2cam["P_rect_0%d" % cam].reshape(3, 4)
    H, W = (int(s) for s in cam2cam["S_rect_02"][::-1].astype(np.int32))
    return np.dot(np.dot(P_rect, R_cam2rect), Rt), (H, W)


def _fmt(a):
    return " ".join("%.6e" % v for v in np.asarray(a, f64).reshape(-1))


def calib_texts(rng, size, toy=None):
    """(calib_cam_to_cam.txt, calib_velo_to_cam.txt) of KITTI's format for rectified size (W, H): plausible values
    drawn from rng, or with toy=(T_z) small integer entries (focal 2, centre (3, 2), no rotation)"""
    W, H = size
    if toy is not None:
        R_rect, R = np.eye(3), np.array([[0, -1, 0], [0, 0, -1], [1, 0, 0]], f64)
        T = np.array([0, 0, toy], f64)
        P2 = np.array([[2, 0, 3, 0], [0, 2, 2, 0], [0, 0, 1, 0]], f64)
        P3 = np.array([[2, 0, 3, -2], [0, 2, 2, 0], [0, 0, 1, 0]], f64)
    else:
        def rot(eps):
            w = rng.uniform(-eps, eps, 3)
            K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
            return np.eye(3) + K + K @ K / 2
        R_rect = rot(0.01)
        R = rot(0.01) @ np.array([[0, -1, 0], [0, 0, -1], [1, 0, 0]], f64)
        T = np.array([rng.uniform(-0.01, 0.0), rng.uniform(-0.08, -0.05), rng.uniform(-0.33, -0.26)])
        f = rng.uniform(700, 730)
        cx, cy = W / 2 + rng.uniform(-15, 15), H / 2 + rng.uniform(-10, 10)
        P2 = np.array([[f, 0, cx, f * 0.06], [0, f, cy, rng.uniform(-0.5, 0.5)], [0, 0, 1, 0.0027]])
        P3 = np.array([[f, 0, cx, -f * 0.47], [0, f, cy, rng.uniform(-3, 3)], [0, 0, 1, 0.0048]])
    cam = ["calib_time: 09-Jan-2012 13:57:47", "corner_dist: 9.950000e-02"]
    for c in range(4):
        Pc = P3 if c == 3 else P2 if c == 2 else np.hstack([P2[:, :3], np.zeros((3, 1))])
        cam += ["S_%02d: %s" % (c, _fmt([1392, 512])), "K_%02d: %s" % (c, _fmt(Pc[:, :3])),
                "D_%02d: %s" % (c, _fmt([-0.37, 0.2, 0.001, 0.001, -0.07])), "R_%02d: %s" % (c, _fmt(np.eye(3))),
                "T_%02d: %s" % (c, _fmt([0.06 * c, 0, 0])), "S_rect_%02d: %s" % (c, _fmt(size)),
                "R_rect_%02d: %s" % (c, _fmt(R_rect)), "P_rect_%02d: %s" % (c, _fmt(Pc))]
    velo = ["calib_time: 15-Mar-2012 11:37:16", "R: %s" % _fmt(R), "T: %s" % _fmt(T),
            "delta_f: %s" % _fmt([0, 0]), "delta_c: %s" % _fmt([0, 0])]
    return "\n".join(cam) + "\n", "\n".join(velo) + "\n"


# five calibration dates (the Eigen test split's, with their rectified sizes) and toy calibrations of small images
DATES = {"2011_09_26": (1242, 375), "2011_09_28": (1224, 370), "2011_09_29": (1238, 374), "2011_09_30": (1226, 370),
         "2011_10_03": (1241, 376)}
TOYS = {"toy": ((8, 6), 0.0), "toy_back": ((8, 6), -1.0), "toy_h1": ((8, 1), 0.0), "toy_w1": ((1, 6), 0.0)}


def make_calibs(seed=2011):
    """{name: (cam_to_cam text, velo_to_cam text)} for DATES and TOYS"""
    rng = np.random.default_rng(seed)
    out = {name: calib_texts(rng, size) for name, size in DATES.items()}
    out.update({name: calib_texts(rng, size, toy=tz) for name, (size, tz) in TOYS.items()})
    return out


def write_calib(dir_, texts):
    os.makedirs(dir_, exist_ok=True)
    for name, text in zip(("calib_cam_to_cam.txt", "calib_velo_to_cam.txt"), texts):
        with open(os.path.join(dir_, name), "w") as f:
            f.write(text)


# ----------------------------------------------------------------------------------------------------- scans
def on_pixel(P, x, u, v):
    """(y, z) of the point at forward distance x whose projection is (u, v) (image coordinates before rint - 1):
    (P0 - u P2) . X = (P1 - v P2) . X = 0 solved for y and z"""
    A = np.array([P[0] - u * P[2], P[1] - v * P[2]], f64)
    rhs = -(A[:, 0] * x + A[:, 3])
    return np.linalg.solve(A[:, 1:3], rhs)


def synthetic_scan(seed, rings=64, per_ring=1900):
    """a seeded (rings x per_ring, 4) float32 scan shaped like a 64-ring scanner's (sensor 1.73 m above a ground
    plane, rings from +2 to -24.9 degrees, clutter in front of the ground, reflectance in [0, 1)); only correctly
    rounded arithmetic, so every machine makes the same bits"""
    rng = np.random.default_rng(seed)
    n = rings * per_ring
    slope = np.repeat(np.linspace(0.035, -0.465, rings), per_ring) + rng.uniform(-1e-3, 1e-3, n)
    t = rng.uniform(-1, 1, n)                              # tan(azimuth / 2) over a half turn, mirrored for the rest
    c, s = (1 - t * t) / (1 + t * t), 2 * t / (1 + t * t)
    c = np.where(rng.random(n) < 0.5, -c, c)
    ground = np.where(slope < 0, 1.73 / -np.minimum(slope, -1e-3), 80.0)
    r = np.minimum(ground, 80.0) * (1 + rng.uniform(-0.01, 0.01, n))
    clutter = rng.random(n) < 0.3
    r = np.where(clutter, rng.uniform(0.05, 1.0, n) * r, r)
    r = np.maximum(r, 0.5)
    pts = np.stack([r * c, r * s, r * slope, rng.random(n)], 1)
    return pts.astype(f32)


def small_scan(seed, n):
    """a seeded scan of n points (the first n of a full-size scan's shape, thinned)"""
    pts = synthetic_scan(seed)
    keep = np.random.default_rng(seed + 1).permutation(pts.shape[0])[:n]
    return pts[np.sort(keep)]


# ----------------------------------------------------------------------------------------------------- data trees
def e2e_frames():
    """the fake Eigen split of the end-to-end fixture: (date, drive, frame, scan seed, points) per line, five dates"""
    out = []
    for k, date in enumerate(sorted(DATES)):
        for j in range(2 if k % 2 == 0 else 1):
            out.append((date, "%s_drive_%04d_sync" % (date, 1 + k), 5 * j + k, 700 + 10 * k + j, 6000 + 1000 * j))
    return out


def write_tree(root, calibs, frames=None):
    """a KITTI raw tree with the frames' calibrations and velodyne scans; returns the split's lines"""
    lines = []
    for date, drive, frame, seed, n in frames or e2e_frames():
        write_calib(os.path.join(root, date), calibs[date])
        d = os.path.join(root, date, drive, "velodyne_points", "data")
        os.makedirs(d, exist_ok=True)
        small_scan(seed, n).tofile(os.path.join(d, "%010d.bin" % frame))
        lines.append("%s/%s %010d l" % (date, drive, frame))
    return lines


def benchmark_depth_png(seed, size):
    """a seeded uint16 KITTI depth PNG's pixels (value = depth x 256, 0 where no depth) of (W, H) size"""
    rng = np.random.default_rng(seed)
    W, H = size
    a = (rng.random((H, W)) * 80 * 256).astype(np.uint16)
    a[rng.random((H, W)) < 0.98] = 0
    return a


def write_benchmark_tree(root, frames=None):
    """eigen_benchmark's proj_depth/groundtruth/image_02 PNGs for the frames; returns the split's lines"""
    from PIL import Image
    lines = []
    for date, drive, frame, seed, _ in frames or e2e_frames():
        d = os.path.join(root, date, drive, "proj_depth", "groundtruth", "image_02")
        os.makedirs(d, exist_ok=True)
        Image.fromarray(benchmark_depth_png(seed, DATES[date])).save(os.path.join(d, "%010d.png" % frame))
        lines.append("%s/%s %010d l" % (date, drive, frame))
    return lines
