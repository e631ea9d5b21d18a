"""GPU parity of k_distribute across node capacities, bit for bit against the CPU oracle (tests marked gpu).

The node capacity M (the largest per-level quota + 4, rounded up to 32) sizes k_distribute's shared memory. The cases cover the two smallest
capacities (M = 32 and 64, at 8 levels and at 1 level), M = 96, and a node list several times the CTA's 256 threads, so the cull compacts
several chunks and each thread of a scan covers several entries. Each case runs a batch of frames on the warp path and on caller canvases."""
import numpy as np
import pytest

from cubemapslam_b200 import config, synth

pytestmark = pytest.mark.gpu

BATCH = 3
CASES = [  # geometry, pyramid levels, nfeatures: M
    ("lafida", 8, 100),     # M = 32
    ("lafida", 8, 250),     # M = 64
    ("lafida", 1, 20),      # M = 32
    ("lafida", 1, 50),      # M = 64
    ("lafida", 8, 300),     # M = 96
    ("front", 8, 12000),    # M = 2624, level 0 keeps more than 3 x 256 key points
]


def _cfg(geom, nlevels, nfeatures):
    kw = {"ORBextractor_nLevels": nlevels, "ORBextractor_nFeatures": nfeatures, "ORBextractor_scaleFactor": 1.2}
    if geom == "front":
        return config.camera("front_cam_params", Camera_Ih=1024, Camera_v0=512.0, CubeFace_w=650, CubeFace_h=650, **kw), \
            config.load_mask("gray_cubemap_front_mask_650")
    return config.camera("lafida_cam0_params", CubeFace_w=450, CubeFace_h=450, **kw), config.load_mask("gray_lafida_cubemap_mask_450")


def _same(got, ref, what):
    for f, ((gk, gd), (rk, rd)) in enumerate(zip(got, ref)):
        assert len(gk) == len(rk) > 0, "%s, frame %d: %d vs %d key points" % (what, f, len(gk), len(rk))
        assert np.array_equal(gk.view(np.uint8), rk.view(np.uint8)), "%s, key points of frame %d" % (what, f)
        assert np.array_equal(gd, rd), "%s, descriptors of frame %d" % (what, f)


@pytest.mark.parametrize("geom,nlevels,nfeatures", CASES)
def test_distribute_node_capacity(oracle, geom, nlevels, nfeatures):
    from cubemapslam_b200.frontend import FrontEnd
    cfg, mask = _cfg(geom, nlevels, nfeatures)
    face = int(cfg["CubeFace.w"])
    cp = oracle.cam_params(cfg)
    m1, m2 = oracle.build_maps(cp)
    ex = oracle.ORBextractor(nfeatures, 1.2, nlevels, 20, 7, face, face)
    frames = np.stack([synth.fisheye_frame(cfg, i) for i in range(2 * BATCH)])
    canvases = np.stack([oracle.warp(cp, fr, m1, m2) for fr in frames])
    canvases[BATCH:, :face, :face] = np.random.default_rng(nfeatures).integers(0, 256, (BATCH, face, face), dtype=np.uint8)
    ref = [ex(c, mask) for c in canvases]
    if nfeatures >= 12000:
        assert max(np.bincount(k["octave"]).max() for k, _ in ref) > 3 * 256
    fe = FrontEnd(cfg, mask, max_batch=BATCH)
    try:
        _same(fe.run(frames[:BATCH]), ref[:BATCH], "warp path")
        _same(fe.extract(canvases[BATCH:]), ref[BATCH:], "caller canvases")   # textured corner face: culled as UNKNOWN_FACE
    finally:
        fe.close()
