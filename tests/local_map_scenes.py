"""Scenes for the local-map SearchByProjection past 4096 MapPoints (cslam_search_by_projection_local_large): one frame of up to 4096 key points
on all five faces and a local map of n MapPoints carrying what Frame::isInFrustum leaves in them. Shared by the oracle-vs-reference test on the
CPU, the GPU test and tools/local_map_latency.py.

What the scenes hold, and why:
- clusters: groups of MapPoints (hundreds in all, most with observations) share one projection, level and descriptor, and their window holds 20
  planted key points at distances 5, 10, ..., 100 on alternating levels, with feature indices in no relation to their positions. Each observed
  member takes the best free one, so dependency chains run through the whole map, and after LM_K (8) members the first stored candidates of
  the rest are all taken while more remain: the commit's fallback. Members sit at indices 4090-4105 and 65530-65545 where those exist.
- two clusters lie on face seams, so their windows cross them in area_cells' swapped / reversed order;
- every planted window also holds two key points with the same descriptor on different levels (equal distances at different visiting
  positions: which one is best decides which slot is taken);
- the rest of the map projects near a random key point with a descriptor a few bits from its own: best and second best at one level on both
  sides of the ratio test, slots overwritten by MapPoints without observations and taken later by observed ones;
- f_taken slots, in_view = 0 rows, view cosines on both sides of 0.998 (float(0.998) itself included), and garbage in every row past a count."""
import numpy as np

from oracle.oracle import KP_DTYPE
from tests import test_gpu_tracking_limits as L

F32 = np.float32
NLEVELS = {8: 1.2, 12: 1.1}          # pyramid levels -> scale factor
CLUSTER_AT = (4090, 65530)           # map indices where cluster members are forced (when the map is that large)
FACES = ((1, 1), (0, 1), (2, 1), (1, 0), (1, 2))   # face origins in units of W: front, left, right, upper, lower


def _flip(rng, d, nbits):
    """d with nbits distinct bits flipped (per row)."""
    d = d.copy()
    for r in range(len(d)):
        for b in rng.choice(256, int(nbits[r]), replace=False):
            d[r, b >> 3] ^= np.uint8(1 << (b & 7))
    return d


def _noise(rng, d, ands):
    """d with every bit flipped with probability 2**-ands."""
    m = rng.integers(0, 256, d.shape, dtype=np.uint8)
    for _ in range(ands - 1):
        m &= rng.integers(0, 256, d.shape, dtype=np.uint8)
    return d ^ m


def _on_face(rng, W, n, face=None):
    f = rng.integers(0, 5, n) if face is None else np.full(n, face)
    o = np.array(FACES)[f] * W
    return (o[:, 0] + rng.uniform(1, W - 1, n)).astype(F32), (o[:, 1] + rng.uniform(1, W - 1, n)).astype(F32)


def frame(seed, W, nkp=4096, nlevels=8):
    """Key points k (cv::KeyPoint records), descriptors d, the planted windows (centre, level, descriptor) and taken slots."""
    rng = np.random.default_rng(900 + seed)
    x, y = _on_face(rng, W, nkp)
    octave = rng.integers(0, nlevels, nkp).astype(np.int32)
    base = rng.integers(0, 256, (48, 32), dtype=np.uint8)
    d = _noise(rng, base[rng.integers(0, 48, nkp)], 7)
    # planted windows: 6 on face interiors, 2 across seams (front/right at x = 2W, front/upper at y = W), and one for each run of members at
    # CLUSTER_AT only, so that the MapPoints past 4095 and past 65535 find free key points
    centres = [(float(cx[0]), float(cy[0])) for cx, cy in (_on_face(rng, W, 1, f) for f in rng.integers(0, 5, 8))]
    centres = centres[:6] + [(2.0 * W - 6, 1.5 * W), (1.5 * W, 1.0 * W + 6)] + centres[6:]
    plants = []
    free = rng.permutation(nkp)
    used = 0
    for ci, (cx, cy) in enumerate(centres):
        lvl = int(rng.integers(nlevels - 2, nlevels))   # windows of at least 10.3 px at th = 1 (members have view cosine 0.5)
        desc = rng.integers(0, 256, 32, dtype=np.uint8)
        idx = free[used:used + 22]; used += 22
        # on a ring of radius ~9.5 px: wider than a grid cell (9 px at face 450, 13 at 650), so no cell holds more than the 16 passing key
        # points the window walk takes per cell
        ang = rng.permutation(22) * (2 * np.pi / 22) + rng.uniform(0, 0.1, 22); rad = rng.uniform(9.3, 9.7, 22)
        x[idx] = (cx + rad * np.cos(ang)).astype(F32); y[idx] = (cy + rad * np.sin(ang)).astype(F32)
        octave[idx[:20]] = np.where(np.arange(20) % 2 == 0, lvl, lvl - 1)
        d[idx[:20]] = _flip(rng, np.repeat(desc[None], 20, 0), 5 * (np.arange(20) + 1))
        octave[idx[20:]] = (lvl, lvl - 1); d[idx[20]] = d[idx[21]] = _flip(rng, desc[None], [7])[0]   # a tie at two visiting positions
        plants.append((F32(cx), F32(cy), lvl, desc))
    keep = np.array([L.ref_safe(a, b, W) for a, b in zip(x, y)])
    x[~keep], y[~keep] = x[~keep] - F32(0.5), y[~keep] - F32(0.5)   # move a cell corner back onto the key point's face
    keep = np.array([L.ref_safe(a, b, W) for a, b in zip(x, y)])
    x[~keep], y[~keep] = _on_face(rng, W, int((~keep).sum()), 0)
    k = np.zeros(nkp, KP_DTYPE); k["x"] = x; k["y"] = y; k["size"] = 31; k["angle"] = rng.uniform(0, 360, nkp).astype(F32); k["octave"] = octave
    taken = (rng.random(nkp) < 0.04).astype(np.uint8)
    return dict(k=k, d=d, taken=taken, plants=plants, planted=free[:used], W=W, nlevels=nlevels, factor=NLEVELS[nlevels])


def local_map(fr, n, seed, stride=None):
    """n MapPoints for frame fr (rows past n up to stride: garbage). Arrays in_view, proj, level, vcos, dq, obs."""
    rng = np.random.default_rng(5000 + seed)
    stride = n if stride is None else stride
    k, d, nl = fr["k"], fr["d"], fr["nlevels"]
    pool = np.setdiff1d(np.arange(len(k)), fr["planted"])
    a = pool[rng.integers(0, len(pool), n)]
    proj = np.stack([k["x"][a], k["y"][a]], 1).astype(F32) + rng.uniform(-2, 2, (n, 2)).astype(F32)
    level = np.clip(k["octave"][a] + rng.integers(0, 2, n), 0, nl - 1).astype(np.int32)
    dq = _noise(rng, d[a], 4)
    in_view = (rng.random(n) < 0.9).astype(np.uint8)
    obs = (rng.random(n) < 0.7).astype(np.uint8)
    vcos = rng.choice(np.array([0.9999, F32(0.998), np.nextafter(F32(0.998), F32(1)), 0.99, 0.5], F32), n)
    # cluster members: 3 % of the map, plus runs at the forced indices
    members = np.nonzero(rng.random(n) < 0.03)[0]
    for s0 in CLUSTER_AT:
        members = np.union1d(members, np.arange(s0, min(n, s0 + 16)))
    members = members[members < n]
    shared = len(fr["plants"]) - len(CLUSTER_AT)
    pc = rng.integers(0, shared, len(members))
    pc[:min(len(members), 40)] = 0   # one cluster of at least 40 members
    for i, s0 in enumerate(CLUSTER_AT):
        pc[(members >= s0) & (members < s0 + 16)] = shared + i
    for m, c in zip(members, pc):
        cx, cy, lvl, desc = fr["plants"][c]
        proj[m] = (cx, cy); level[m] = lvl; dq[m] = desc; in_view[m] = 1; vcos[m] = 0.5; obs[m] = rng.random() < 0.85
    out = dict(in_view=in_view, proj=proj, level=level, vcos=vcos, dq=dq, obs=obs)
    if stride > n:   # garbage past the count, including levels no search could take
        g = stride - n
        extra = dict(in_view=np.ones(g, np.uint8), proj=rng.uniform(-1e4, 1e4, (g, 2)).astype(F32), level=rng.integers(-50, 50, g).astype(np.int32),
                     vcos=rng.uniform(-2, 2, g).astype(F32), dq=rng.integers(0, 256, (g, 32), dtype=np.uint8), obs=rng.integers(0, 256, g).astype(np.uint8))
        out = {key: np.concatenate([out[key], extra[key]]) for key in out}
    return out


def scales(nlevels):
    return L.level_tables(nlevels, NLEVELS[nlevels])[0]


def oracle_search(oracle, fr, mp, n, th, nn):
    """The oracle's answer on the first n rows of map mp."""
    g = oracle.FrameGrid(fr["k"], fr["W"], fr["W"])
    return g.search_by_projection_local(fr["d"], scales(fr["nlevels"]), mp["in_view"][:n], mp["proj"][:n], mp["level"][:n], mp["vcos"][:n], mp["dq"][:n],
                                        mp["obs"][:n].astype(np.int32), fr["taken"], th, nn)
