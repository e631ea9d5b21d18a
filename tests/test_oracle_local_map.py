"""The oracle's local-map SearchByProjection (oracle/frame_index.h) against the reference's own CPU body (ref_search_by_projection_local in
oracle/ref_api.cpp, on reference Frame / MapPoint objects) at 4097, 16 384 and 65 537 MapPoints, face sizes 450 and 650, th 1 and 5: the sizes
cslam_search_by_projection_local_large takes past the 4096 of cslam_search_by_projection_local. The reference's answers are recorded in
tests/golden/refcalls_oracle_local_map.npz, so the test also runs where oracle/_ref cannot be built."""
import numpy as np
import pytest

from cubemapslam_b200 import config
from oracle import ref

from . import local_map_scenes as S
from .refrecord import LIVE, RefRecord, same
from .test_oracle_projection import CAMS

REC = RefRecord("oracle_local_map")
NN = 0.8


@pytest.fixture(scope="module", params=(450, 650))
def cam(request, oracle):
    W = request.param
    c = dict(CAMS[W]); name = c.pop("name")
    return W, ref.Ref(oracle.cam_params(config.camera(name, **c))) if LIVE else None


@pytest.mark.parametrize("n", (4097, 16384, 65537))
@pytest.mark.parametrize("th", (1.0, 5.0))
def test_local_map_oracle_vs_reference(oracle, cam, n, th):
    W, r = cam
    fr = S.frame(W + n, W)
    mp = S.local_map(fr, n, n + int(th))
    on, om = S.oracle_search(oracle, fr, mp, n, th, NN)

    def run():
        rn, rm = r.search_by_projection_local(fr["k"], fr["d"], mp["in_view"], mp["proj"], mp["level"], mp["vcos"], mp["dq"], mp["obs"].astype(np.int32), fr["taken"], th, NN)
        return rn, np.where(rm == -2, -1, rm)   # -2: a slot that held a MapPoint before the call (f_taken) and still does
    rn, rm = REC("local_%d_%d_%d" % (W, n, th), run)
    assert on == rn > 0 and same(np.asarray(om, np.int32), rm)
    assert (om >= 4096).any()
    if n > 65536:
        assert (om >= 65536).any()
