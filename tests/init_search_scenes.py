"""Scenes for SearchForInitialization (cslam_search_for_initialization, the oracle's fi_search_for_initialization and the reference's own
body), shared by the oracle-vs-reference test on the CPU, the GPU test and tools/init_search_latency.py. Every scene is (k1, d1, k2, d2, xy):
F1's and F2's key points and descriptors and the window centres (vbPrevMatched). Every key point lies on a face, 1 px or more from its seams,
and passes the reference's PosInGrid check, so the reference's own Frames can hold them.

- extracted(W): the initialisation extractor's frames (3 * nFeatures features: 6000 at face 450, 9000 at face 650) of a synthetic fisheye
  frame, F2 the same canvas shifted by a few pixels with noise (a perturbed view); centres = F1's key points, as Tracking starts.
- chain(W): F1 and three successive perturbed views, for calls that carry vbPrevMatched forward.
- dense(seed, W, n1, n2): clusters of key points of every octave around a few centres, descriptors a few bits from four bases (equal
  distances at different visiting positions, candidates whose vMatchedDistance equals their distance, later queries taking earlier ones' key
  points), windows of more than 256 candidates and 13-px cells of more than 16 level-0 key points, windows across face seams, centres on
  corner tiles and outside the canvas.
- steal(): a later query takes an earlier one's key point, and the earlier one's stale rotation-bin entry changes the three maxima so that
  the later match is cleared."""
import numpy as np

from cubemapslam_b200 import config, synth
from oracle import init_search
from oracle.oracle import KP_DTYPE
from tests import test_gpu_tracking_limits as L

F32 = np.float32
FACES = ((1, 1), (0, 1), (2, 1), (1, 0), (1, 2))   # face origins in units of W: front, left, right, upper, lower
CAMS = {333: dict(name="front_cam_params", Camera_Ih=1024, Camera_v0=512.0, CubeFace_w=333, CubeFace_h=333),
        450: dict(name="lafida_cam0_params", CubeFace_w=450, CubeFace_h=450),
        650: dict(name="front_cam_params", Camera_Ih=1024, Camera_v0=512.0)}
EXTRACTED = {450: 6000, 650: 9000}    # 3 * nFeatures of the initialisation extractor


def cam_cfg(W):
    c = dict(CAMS[W]); name = c.pop("name")
    return config.camera(name, **c)


def _safe(k, W):
    keep = np.array([L.ref_safe(x, y, W) and min((x % W), (y % W)) >= 1 and max((x % W), (y % W)) <= W - 1 for x, y in zip(k["x"], k["y"])], bool)
    return keep


def _extract(oracle, W, canvas):
    mask = config.load_mask("gray_lafida_cubemap_mask_450") if W == 450 else np.full((3 * W, 3 * W), 255, np.uint8)
    k, d = oracle.ORBextractor(EXTRACTED[W], 1.2, 8, 20, 7, W, W)(canvas, mask)
    keep = _safe(k, W)
    return np.ascontiguousarray(k[keep]), np.ascontiguousarray(d[keep])


def _views(oracle, W, nviews):
    cfg = cam_cfg(W); cp = oracle.cam_params(cfg)
    m1, m2 = oracle.build_maps(cp)
    canvas = oracle.warp(cp, synth.fisheye_frame(cfg, 4), m1, m2).astype(np.int16)
    rng = np.random.default_rng(W)
    out = []
    for v in range(nviews):
        c = np.roll(canvas, (2 * v, 3 * v), axis=(0, 1)) + (rng.integers(-2, 3, canvas.shape) if v else 0)
        out.append(_extract(oracle, W, np.clip(c, 0, 255).astype(np.uint8)))
    return out


def extracted(oracle, W):
    (k1, d1), (k2, d2) = _views(oracle, W, 2)
    return k1, d1, k2, d2, np.stack([k1["x"], k1["y"]], 1).astype(F32)


def chain(oracle, W, nviews=4):
    return _views(oracle, W, nviews)


def _flip(rng, d, nbits):
    d = d.copy()
    for r in range(len(d)):
        for b in rng.choice(256, int(nbits[r]), replace=False):
            d[r, b >> 3] ^= np.uint8(1 << (b & 7))
    return d


def _cluster_points(rng, W, centres, n, spread):
    c = centres[rng.integers(0, len(centres), n)]
    x = c[:, 0] + rng.normal(0, spread, n); y = c[:, 1] + rng.normal(0, spread, n)
    return x.astype(F32), y.astype(F32)


def _keypoints(rng, W, n, centres, spread, nlevels=8):
    k = np.zeros(n, KP_DTYPE)
    filled = 0
    while filled < n:
        x, y = _cluster_points(rng, W, centres, 2 * (n - filled) + 16, spread)
        ok = _safe(np.rec.fromarrays([x, y], names="x,y"), W)
        x, y = x[ok][:n - filled], y[ok][:n - filled]
        k["x"][filled:filled + len(x)] = x; k["y"][filled:filled + len(y)] = y
        filled += len(x)
    k["octave"] = np.where(rng.random(n) < 0.6, 0, rng.integers(1, nlevels, n))
    k["angle"] = np.mod(rng.choice(np.array([3.0, 27.0, 95.0, 181.0, 335.5], F32), n) + rng.integers(0, 3, n).astype(F32) * F32(12), F32(360))   # [0, 360) as cv::KeyPoint
    k["size"] = 31; k["class_id"] = -1
    return k


def dense(seed, W, n1, n2):
    rng = np.random.default_rng(7000 + seed)
    # cluster centres: face interiors, and on both sides of the front face's seams so that windows cross them
    centres = [(o[0] * W + W * 0.5, o[1] * W + W * 0.5) for o in FACES] + [(2 * W - 20, 1.5 * W), (1.5 * W, W + 15), (W + 25, 1.5 * W), (1.5 * W, 2 * W - 30),
                                                                         (1.5 * W, 0.5 * W), (2.5 * W, 1.5 * W + 0.4 * W)]
    centres = np.array(centres, np.float64)
    k2 = _keypoints(rng, W, n2, centres, 25.0)
    if n2 >= 100:   # 40 level-0 key points in a 3-px box: one grid cell holds more than 16 of them
        k2["x"][:40] = F32(centres[0, 0] + 0.3) + rng.uniform(0, 3, 40).astype(F32); k2["y"][:40] = F32(centres[0, 1] + 0.3) + rng.uniform(0, 3, 40).astype(F32)
        k2["octave"][:40] = 0
    k1 = _keypoints(rng, W, n1, centres, 30.0)
    base = rng.integers(0, 256, (4, 32), dtype=np.uint8)
    d2 = _flip(rng, base[rng.integers(0, 4, n2)], rng.integers(0, 4, n2))
    d1 = _flip(rng, base[rng.integers(0, 4, n1)], rng.integers(0, 30, n1))
    xy = np.stack([k1["x"], k1["y"]], 1).astype(F32) + rng.normal(0, 3, (n1, 2)).astype(F32)
    # some centres on a corner tile, outside the canvas, or exactly on a key point of F2
    m = rng.random(n1)
    xy[m < 0.02] = (F32(0.5 * W), F32(0.5 * W))
    xy[(m >= 0.02) & (m < 0.03)] = (F32(-5), F32(4 * W))
    on = (m >= 0.03) & (m < 0.08)
    xy[on] = np.stack([k2["x"], k2["y"]], 1)[rng.integers(0, max(n2, 1), on.sum())] if n2 else xy[on]
    return k1, d1, k2, d2, np.ascontiguousarray(xy)


def steal(W=650):
    """Queries in F1 order: two pairs in bins 1 and 2, then q0 -> X (distance 40, bin 5), then q1 -> X (distance 20, bin 7), which takes X
    from q0. Bin sizes 2, 2, 1 (q0, stale), 1: the three maxima are bins 1, 2 and 5, so q1's match is cleared, and 4 matches remain."""
    rng = np.random.default_rng(5)
    spots = [(W + 100 + 180 * (i % 3), W + 100 + 200 * (i // 3)) for i in range(5)]   # 180+ px apart: each window holds one F2 key point
    k2 = np.zeros(5, KP_DTYPE); k1 = np.zeros(6, KP_DTYPE)
    d2 = rng.integers(0, 256, (5, 32), dtype=np.uint8)
    for i, (x, y) in enumerate(spots):
        k2[i]["x"], k2[i]["y"], k2[i]["angle"] = x, y, 1.0
    # F1: (spot, bits flipped, bin)
    plan = [(0, 5, 1), (1, 6, 1), (2, 7, 2), (3, 8, 2), (4, 40, 5), (4, 20, 7)]
    d1 = np.zeros((6, 32), np.uint8)
    for i, (s, bits, b) in enumerate(plan):
        k1[i]["x"], k1[i]["y"] = spots[s][0] + 1, spots[s][1] + 1
        k1[i]["angle"] = 1.0 + 12.0 * b
        d1[i] = _flip(rng, d2[s:s + 1], [bits])[0]
    for k in (k1, k2):
        k["size"] = 31; k["class_id"] = -1
    return k1, d1, k2, d2, np.stack([k1["x"], k1["y"]], 1).astype(F32)


def oracle_search(scene, W, window_size=100, nnratio=0.9, check_ori=True):
    return init_search.search(*scene, W, window_size, nnratio, check_ori)
