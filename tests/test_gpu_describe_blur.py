"""k_describe's blur and BRIEF against the oracle's ORBextractor, bit for bit, on caller canvases built to reach its corner cases.

The 7x7 blur is exact in integers: H = sum g P <= 65280 per row, dst = (sum g H + 32768) >> 16 with g = [18,34,48,56,48,34,18]. The
canvases here put key points where that arithmetic is at its limits:
- large saturated blocks at 255 next to texture, so whole rows of a patch reach H = 65280 (high byte 255);
- row and column steps of 64 grey levels, where sum g H lands exactly on a rounding boundary (V = 65536 k + 32768);
- key points at every patch offset x mod 16 (the interior patch copy starts at a 16-byte boundary);
- key points within 21 px of every level edge, where the patch is read with REFLECT_101.
The coverage of each case is checked on the oracle's key points without a GPU; the parity tests compare the GPU with the oracle."""
import numpy as np
import pytest

from cubemapslam_b200 import config

FACE, SCALE, NLEVELS, NFEATURES = 333, 1.2, 8, 3000
G7 = np.array([18, 34, 48, 56, 48, 34, 18], np.int64)


def _cfg():
    return config.camera("lafida_cam0_params", CubeFace_w=FACE, CubeFace_h=FACE, ORBextractor_scaleFactor=SCALE,
                         ORBextractor_nLevels=NLEVELS, ORBextractor_nFeatures=NFEATURES)


def _canvas(seed):
    """Blocks of 24-40 px: saturated (255), flat at a multiple of 64, random texture, or steps of 64 along rows or columns."""
    rng = np.random.default_rng(seed)
    n = 3 * FACE
    c = np.empty((n, n), np.uint8)
    y = 0
    while y < n:
        bh = int(rng.integers(24, 41))
        x = 0
        while x < n:
            bw = int(rng.integers(24, 41))
            blk = c[y:y + bh, x:x + bw]
            kind = rng.integers(0, 5)
            if kind == 0:
                blk[:] = 255
            elif kind == 1:
                blk[:] = 64 * int(rng.integers(0, 4))
            elif kind == 2:
                blk[:] = rng.integers(0, 256, blk.shape)
            elif kind == 3:   # steps of 64 down the rows
                blk[:] = (64 * ((np.arange(blk.shape[0]) // int(rng.integers(1, 5))) % 4) + int(rng.integers(0, 2)) * 63)[:, None]
            else:             # steps of 64 along the columns
                blk[:] = (64 * ((np.arange(blk.shape[1]) // int(rng.integers(1, 5))) % 4) + int(rng.integers(0, 2)) * 63)[None, :]
            x += bw
        y += bh
    return c


def _hv(img):
    """H and V of the fixed-point blur (REFLECT_101), as int64."""
    p = np.pad(img.astype(np.int64), 3, mode="reflect")
    h = sum(G7[t] * p[:, t:t + img.shape[1]] for t in range(7))
    return h, sum(G7[t] * h[t:t + img.shape[0], :] for t in range(7))


def _level_coords(kps, ex):
    """Level pixel of each key point: kp.x = lx * scale of its octave, rounded in fp32."""
    oct_ = kps["octave"]
    s = ex.scale[oct_]
    lx = np.rint(kps["x"] / s).astype(np.int64)
    ly = np.rint(kps["y"] / s).astype(np.int64)
    assert np.array_equal(np.float32(lx) * s, kps["x"]) and np.array_equal(np.float32(ly) * s, kps["y"])
    return oct_, lx, ly


@pytest.fixture(scope="module")
def cases(oracle):
    mask = np.full((3 * FACE, 3 * FACE), 255, np.uint8)
    ex = oracle.ORBextractor(NFEATURES, SCALE, NLEVELS, 20, 7, FACE, FACE)
    out = []
    for seed in range(3):
        canv = _canvas(seed)
        kps, desc = ex(canv, mask)
        lv = [ex.level_image(l) for l in range(NLEVELS)]
        out.append((canv, kps, desc, lv, _level_coords(kps, ex)))
    return mask, out


def test_canvases_reach_every_case(cases):
    """Saturated rows, rounding ties, all 16 patch offsets and all four REFLECT_101 edges occur under the oracle's key points."""
    _, cs = cases
    offsets, edges, sat, ties = set(), set(), 0, 0
    for _, kps, _, lv, (oct_, lx, ly) in cs:
        assert len(kps) > 1000
        for l in range(NLEVELS):
            sel = oct_ == l
            if not sel.any():
                continue
            h, w = lv[l].shape
            H, V = _hv(lv[l])
            for x, y in zip(lx[sel], ly[sel]):
                if x >= 21 and y >= 21 and x + 21 < w and y + 21 < h:
                    offsets.add(int((x - 21) % 16))
                    rows = H[y - 21:y + 22, x - 18:x + 19]   # the H values the 37 blurred columns of this patch use
                    sat += int((rows == 65280).all(axis=1).any())
                    ties += int(((V[y - 18:y + 19, x - 18:x + 19] & 0xffff) == 32768).any())
                edges |= {e for e, hit in (("left", x < 21), ("top", y < 21), ("right", x + 21 >= w), ("bottom", y + 21 >= h)) if hit}
    assert offsets == set(range(16)), sorted(offsets)
    assert edges == {"left", "top", "right", "bottom"}, edges
    assert sat > 50, sat
    assert ties > 50, ties


@pytest.mark.gpu
def test_describe_blur_cases(cases):
    from cubemapslam_b200.frontend import FrontEnd
    mask, cs = cases
    fe = FrontEnd(_cfg(), mask, max_batch=len(cs))
    try:
        res = fe.extract(np.stack([c[0] for c in cs]))
        for f, (_, kps, desc, _, _) in enumerate(cs):
            gk, gd = res[f]
            assert len(gk) == len(kps), "canvas %d: %d vs %d key points" % (f, len(gk), len(kps))
            assert np.array_equal(gk.view(np.uint8), kps.view(np.uint8)), "key points, canvas %d" % f
            bad = np.nonzero((gd != desc).any(axis=1))[0]
            assert len(bad) == 0, "canvas %d: %d descriptors differ, first at key point %d" % (f, len(bad), bad[0])
    finally:
        fe.close()


@pytest.mark.gpu
def test_describe_blur_one_canvas_per_call(cases):
    """The same canvases one per call (batch 1), so every key point's warp runs with a frame index of 0."""
    from cubemapslam_b200.frontend import FrontEnd
    mask, cs = cases
    fe = FrontEnd(_cfg(), mask, max_batch=1)
    try:
        for f, (canv, kps, desc, _, _) in enumerate(cs):
            gk, gd = fe.extract(canv)
            assert np.array_equal(gk.view(np.uint8), kps.view(np.uint8)) and np.array_equal(gd, desc), "canvas %d" % f
    finally:
        fe.close()
