"""GPU parity of the tiled k_warp and the corner-skipping k_pyramid against the CPU oracle, bit for bit (tests marked gpu).

k_warp stages each 32 x 32 output tile's source box in shared memory (4-byte copies when source rows are word-aligned, byte loads
otherwise) and gathers tiles whose box is too large straight from global memory. k_pyramid on the warp path leaves the provably
black cubemap corners of every level untouched, so those regions must already hold zeros, also after a caller-canvas extract."""
import numpy as np
import pytest

from cubemapslam_b200 import config, synth

pytestmark = pytest.mark.gpu

BATCHES = (1, 3, 5, 13)       # 13: not a multiple of the 4 or 8 frames a k_warp CTA handles
WT, BOX_MAX = 32, 6144        # k_warp tile edge and the largest staged box (bytes), as in frontend.cu


def _cfg(geom, face):
    if geom == "front":   # the benchmark's 1280 x 1024 sensor (config.front_1024) at another face size
        return config.camera("front_cam_params", Camera_Ih=1024, Camera_v0=512.0, CubeFace_w=face, CubeFace_h=face)
    return config.camera("lafida_cam0_params", CubeFace_w=face, CubeFace_h=face)


def _fe(cfg, max_batch):
    from cubemapslam_b200.frontend import FrontEnd
    face = int(cfg["CubeFace.w"])
    return FrontEnd(cfg, np.full((3 * face, 3 * face), 255, np.uint8), max_batch=max_batch)


def _tile_kinds(cp, m1, m2):
    """(staged, direct) k_warp tile counts, by the create-time rule: box of ix..ix+1, iy..iy+1 over the pixels whose map is not (0,0)."""
    W = cp.faceW
    sx = np.rint(m1 * 32).astype(np.int64); sy = np.rint(m2 * 32).astype(np.int64)
    staged = direct = 0
    for tc, tr in ((1, 1), (0, 1), (2, 1), (1, 0), (1, 2)):
        cx0 = tc * W
        for y0 in range(0, W, WT):
            for xa in range(cx0 // WT * WT, cx0 + W, WT):
                a, b = max(xa, cx0), min(xa + WT, cx0 + W)
                X = sx[tr * W + y0:tr * W + min(y0 + WT, W), a:b]; Y = sy[tr * W + y0:tr * W + min(y0 + WT, W), a:b]
                live = (X != 0) | (Y != 0)
                if not live.any():
                    staged += 1
                    continue
                ix, iy = X[live] >> 5, Y[live] >> 5
                bx0 = ix.min() & ~3
                box = (ix.max() + 2 - bx0 + 3) // 4 * 4 * (iy.max() + 2 - iy.min())
                direct += box > BOX_MAX; staged += box <= BOX_MAX
    return staged, direct


@pytest.mark.parametrize("face", [333, 560, 570, 610, 650])
@pytest.mark.parametrize("geom", ["lafida", "front"])
def test_warp_tiles_bit_exact(oracle, geom, face):
    cfg = _cfg(geom, face)
    cp = oracle.cam_params(cfg)
    m1, m2 = oracle.build_maps(cp)
    frames = np.stack([synth.fisheye_frame(cfg, i) for i in range(max(BATCHES))])
    frames[-1, 0, 0] = 200        # the pixels outside the image circle read S(0, 0): make it non-zero in one frame
    ref = [oracle.warp(cp, f, m1, m2) for f in frames]
    fe = _fe(cfg, max(BATCHES))
    try:
        for b in BATCHES:
            got = fe.warp(frames[-b:])
            for i in range(b):
                assert np.array_equal(got[i], ref[len(frames) - b + i]), "%s face %d batch %d frame %d" % (geom, face, b, i)
    finally:
        fe.close()


def test_warp_direct_gather_tiles(oracle):
    """A small face magnifies each 32 x 32 tile's footprint in the fisheye beyond the staging budget: those tiles gather from global."""
    cfg = _cfg("lafida", 96)
    cp = oracle.cam_params(cfg)
    m1, m2 = oracle.build_maps(cp)
    staged, direct = _tile_kinds(cp, m1, m2)
    assert direct > 0 and staged > 0
    frames = np.stack([synth.fisheye_frame(cfg, i) for i in range(5)])
    fe = _fe(cfg, 5)
    try:
        got = fe.warp(frames)
        for i in range(5):
            assert np.array_equal(got[i], oracle.warp(cp, frames[i], m1, m2)), "frame %d" % i
    finally:
        fe.close()


def test_warp_unaligned_device_frames(oracle):
    """Frames at an odd device address: the 4-byte staging copies cannot be used, the byte loads must give the same canvas."""
    import torch
    cfg = config.front_1024()
    cp = oracle.cam_params(cfg)
    m1, m2 = oracle.build_maps(cp)
    frames = np.stack([synth.fisheye_frame(cfg, i) for i in range(3)])
    fe = _fe(cfg, 3)
    try:
        dev = torch.device("cuda", 0)
        buf = torch.zeros(frames.size + 1, dtype=torch.uint8, device=dev)
        buf[1:] = torch.from_numpy(frames.reshape(-1)).to(dev)
        kps = torch.empty((3, fe.kp_cap, 28), dtype=torch.uint8, device=dev); desc = torch.empty((3, fe.kp_cap, 32), dtype=torch.uint8, device=dev)
        n = torch.empty(3, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        fe.run_dev(buf.data_ptr() + 1, 3, kps.data_ptr(), desc.data_ptr(), n.data_ptr())
        fe.sync()
        for i in range(3):
            assert np.array_equal(fe.level_image(i, 0), oracle.warp(cp, frames[i], m1, m2)), "frame %d" % i
    finally:
        fe.close()


@pytest.mark.parametrize("geom,face", [("front", 650), ("lafida", 450), ("lafida", 333)])
def test_pyramid_whole_levels(oracle, geom, face):
    """Every level, corners included, equals the oracle's resize_linear chain over the whole canvas."""
    cfg = config.front_1024() if (geom, face) == ("front", 650) else _cfg(geom, face)
    cp = oracle.cam_params(cfg)
    m1, m2 = oracle.build_maps(cp)
    frames = np.stack([synth.fisheye_frame(cfg, i) for i in range(3)])
    fe = _fe(cfg, 3)
    try:
        fe.run(frames)
        for f in range(3):
            lvl = oracle.warp(cp, frames[f], m1, m2)
            assert np.array_equal(fe.level_image(f, 0), lvl)
            for l in range(1, fe.nlevels):
                h, w = fe.level_image(f, l).shape
                lvl = oracle.resize_linear(lvl, w, h)
                assert np.array_equal(fe.level_image(f, l), lvl), "frame %d level %d" % (f, l)
    finally:
        fe.close()


def test_caller_canvas_then_warp_path(oracle):
    """A caller-canvas extract fills every level's corners; the next warp-path run must clear them all, not just level 0."""
    cfg = config.lafida_450()
    cp = oracle.cam_params(cfg)
    m1, m2 = oracle.build_maps(cp)
    canv = np.stack([oracle.warp(cp, synth.fisheye_frame(cfg, i), m1, m2) for i in range(3)])
    for c in canv:   # flat grey corners: non-zero on every level, but no texture to flood the candidate buffers
        for v, (ty, tx) in zip((37, 90, 150, 220), ((0, 0), (0, 900), (900, 0), (900, 900))):
            c[ty:ty + 450, tx:tx + 450] = v
    frames = np.stack([synth.fisheye_frame(cfg, i) for i in (4, 5, 6)])
    fe = _fe(cfg, 3); fresh = _fe(cfg, 3)
    try:
        fe.extract(canv)
        got = fe.run(frames)
        want = fresh.run(frames)
        for f in range(3):
            for l in range(fe.nlevels):
                assert np.array_equal(fe.level_image(f, l), fresh.level_image(f, l)), "frame %d level %d" % (f, l)
            assert np.array_equal(got[f][0].view(np.uint8), want[f][0].view(np.uint8)) and np.array_equal(got[f][1], want[f][1]), "frame %d" % f
    finally:
        fe.close(); fresh.close()
