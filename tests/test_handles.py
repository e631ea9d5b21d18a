"""The library's handles share one lifecycle (cslam::Handle in csrc/common.cuh, _capi.Handle in Python): layout checks on the sources, the
launches each call counts, and the failure and close paths."""
import glob
import os
import re

import numpy as np
import pytest

from cubemapslam_b200 import _capi, config, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "cubemapslam_b200", "csrc")
HANDLES = {"cslam_frontend", "cslam_matcher", "cslam_vocabulary", "cslam_tracker", "cslam_optimizer", "cslam_mapper"}


def _sources():
    return {os.path.basename(p): open(p).read() for p in glob.glob(os.path.join(CSRC, "*.cu*"))}


def _body(src, head):
    b = src.index(head)
    return src[b:re.compile(r"\n\}").search(src, b).end()]


def test_every_handle_derives_from_the_base():
    found = {}
    for name, src in _sources().items():
        for m in re.finditer(r"\bstruct\s+(cslam_\w+)\s*(?::\s*([\w:]+)\s*)?\{", src):
            found[m.group(1)] = (name, m.group(2))
    assert set(found) == HANDLES, found
    assert all(base == "cslam::Handle" for _, base in found.values()), found


def test_streams_are_created_by_the_base_and_the_front_end_lanes_only():
    srcs = _sources()
    open_body = _body(srcs["capi_common.cu"], "int Handle::open(")
    for name, src in srcs.items():
        for m in re.finditer(r"\bcudaStreamCreate\w*\s*\(", src):
            line = src[src.rfind("\n", 0, m.start()) + 1:src.find("\n", m.start())]
            in_open = name == "capi_common.cu" and m.start() >= src.index(open_body) and m.start() < src.index(open_body) + len(open_body)
            in_lanes = name == "frontend.cu" and "lane[" in line
            assert in_open or in_lanes, "%s: %s" % (name, line.strip())
    assert re.search(r"\bcudaStreamCreate\w*\s*\(", open_body)


def test_no_device_wide_synchronise():
    """A handle waits for its own streams: the GPU is shared with other work."""
    offenders = [name for name, src in _sources().items() if "cudaDeviceSynchronize" in src]
    assert not offenders, offenders


def test_only_capi_declares_return_types():
    """_capi.lib() declares every restype of the library once; no other module sets one."""
    paths = glob.glob(os.path.join(ROOT, "cubemapslam_b200", "*.py")) + glob.glob(os.path.join(ROOT, "tests", "*.py")) + \
        glob.glob(os.path.join(ROOT, "tools", "*.py")) + [os.path.join(ROOT, f) for f in ("bench.py", "bench_extra.py", "__graft_entry__.py")]
    offenders = [os.path.relpath(p, ROOT) for p in paths
                 if os.path.basename(p) != "_capi.py" and re.search(r"\.restype\s*=", open(p).read())]
    assert not offenders, offenders


def _launched(h, call):
    l0 = h.launches
    call()
    return h.launches - l0


@pytest.mark.gpu
def test_mapper_launch_counts():
    from cubemapslam_b200.mapper import Mapper
    s = synth.mapping_pair(0, n=400, faceW=650)
    n = len(s["Xw"])
    level = np.clip(s["kLast"]["octave"], 0, 7).astype(np.int32)
    a, b = len(s["kCur"]), len(s["kLast"])
    m = Mapper()
    try:
        desc = np.random.default_rng(0).integers(0, 256, (10, 32), dtype=np.uint8)
        assert _launched(m, lambda: m.ComputeDistinctiveDescriptors(desc, [0, 4, 10])) == 1
        # the key frame's frame index, then the search
        assert _launched(m, lambda: m.FuseSearch(s["kCur"], s["dCur"], s["TcwCur"], np.ones(n, np.uint8), s["Xw"], level, s["dLast"], 3.0, s["scale"],
                                                 s["inv_level_sigma2"], 650, 650)) == 2
        tri = lambda: m.SearchForTriangulation(s["kCur"][None], s["dCur"][None], np.zeros((1, a, 3), np.float32), s["hasMPCur"][None], s["nodeCur"][None], [a],
                                               s["kLast"][None], s["dLast"][None], np.zeros((1, b, 3), np.float32), s["hasMPObs"][None], s["nodeObs"][None], [b],
                                               np.zeros((1, 3), np.float32), s["TcwLast"].reshape(1, 16), s["E12"].reshape(1, 9), s["scale"], s["level_sigma2"], 650, 650)
        assert _launched(m, tri) == 1
    finally:
        m.close()


@pytest.mark.gpu
def test_tracker_launches_per_host_call():
    from cubemapslam_b200.tracker import Tracker
    s = synth.tracking_pair(0, n=1500, faceW=650)
    cth = np.float32(np.cos(np.radians(95.0)))
    rng = np.random.default_rng(0)
    pick = np.nonzero(s["src"] >= 0)[0][:500]
    proj = np.stack([s["kCur"]["x"][pick], s["kCur"]["y"][pick]], 1).astype(np.float32)
    lvl = s["kCur"]["octave"][pick].astype(np.int32)
    t = Tracker(max_frames=2, max_features=4096)
    try:
        assert _launched(t, lambda: t.frame_index(s["kCur"], 650, 650)) == 1
        # both searches index the current frame first; the local-map search then runs in two launches (candidates, commit)
        assert _launched(t, lambda: t.SearchByProjection_last(s["kCur"], s["dCur"], s["TcwCur"], s["kLast"], s["hasMP"], s["Xw"], s["dLast"], s["mpObs"], s["curTaken"],
                                                              650, 650, cth, 15.0, True)) == 2
        assert _launched(t, lambda: t.SearchByProjection_local(s["kCur"], s["dCur"], np.ones(len(pick), np.uint8), proj, lvl, np.full(len(pick), 0.99, np.float32),
                                                               s["dLast"][s["src"][pick]], np.ones(len(pick), np.int32),
                                                               (rng.random(len(s["kCur"])) < 0.05).astype(np.uint8), 650, 650, 3.0, 0.8)) == 3
    finally:
        t.close()


@pytest.mark.gpu
def test_matcher_and_optimizer_launch_counts():
    from cubemapslam_b200.matcher import ORBMatcher
    from cubemapslam_b200.optimizer import Optimizer
    A, aA, B, aB, _ = synth.descriptor_pair(0, n=256)
    m = ORBMatcher(max_pairs=1, max_features=256)
    o = Optimizer()
    try:
        assert _launched(m, lambda: m.match_bruteforce(A, aA, B, aB)) == 1
        q = synth.pose_problem(n=200, faceW=450, seed=5)
        assert _launched(o, lambda: o.PoseOptimization(q["Tcw"], q["Xw"], q["kpxy"], q["inv_sigma2"], 450, 450)) == 1
    finally:
        m.close()
        o.close()


@pytest.mark.gpu
def test_failed_create_leaves_the_device_usable():
    """The quadtree check fails after the front end's level buffers are allocated: the partly built handle is released, and the next front
    end on the device computes what one created before the failure did."""
    from cubemapslam_b200.frontend import FrontEnd
    cfg = config.lafida_450()
    mask = config.load_mask("gray_lafida_cubemap_mask_450")
    frame = synth.fisheye_frame(cfg, 0)

    def extract():
        fe = FrontEnd(cfg, mask, max_batch=1)
        try:
            return fe.run(frame)
        finally:
            fe.close()
    want = extract()
    with pytest.raises(_capi.CslamError, match="quadtree"):
        FrontEnd(cfg, mask, max_batch=1, orb=_capi.orb_params(cfg, nfeatures=100000))
    got = extract()
    assert len(want[0]) > 0 and np.array_equal(got[0].view(np.uint8), want[0].view(np.uint8)) and np.array_equal(got[1], want[1])


@pytest.mark.gpu
def test_close_twice_is_harmless():
    from cubemapslam_b200.frontend import FrontEnd
    from cubemapslam_b200.mapper import Mapper
    from cubemapslam_b200.matcher import ORBMatcher
    from cubemapslam_b200.optimizer import Optimizer
    from cubemapslam_b200.tracker import Tracker
    from cubemapslam_b200.vocabulary import Vocabulary
    voc = synth.vocabulary(k=6, L=3)
    makers = [lambda: FrontEnd(config.lafida_450(), config.load_mask("gray_lafida_cubemap_mask_450"), max_batch=1), lambda: ORBMatcher(max_pairs=1, max_features=64),
              lambda: Vocabulary(6, 3, voc["parent"], voc["is_leaf"], voc["desc"], voc["weight"], max_frames=1, max_features=64), lambda: Tracker(max_frames=1, max_features=64),
              Optimizer, Mapper]
    for make in makers:
        h = make()
        h.close()
        h.close()
        del h
