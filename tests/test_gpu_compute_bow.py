"""Frame::ComputeBoW / KeyFrame::ComputeBoW on the GPU. cslam_bow_transform_fv (BowVector + FeatureVector, up to 16384 features per frame)
against the oracle, and the drop-in definitions (dropin/ComputeBoW_b200.cpp, linked in oracle/_ref/libdropin_bow.so with the reference's own
Frame / KeyFrame / DBoW2) against the reference's CPU bodies on identical objects."""
import ctypes as C

import numpy as np
import pytest

from cubemapslam_b200 import config
from tests.test_gpu_bow_limits import _noise, unbalanced_tree
from tests.test_oracle_compute_bow import dropin_lib, feature_vector, frame_features, load_vocabulary, write_with_newline

pytestmark = pytest.mark.gpu
STRIDE = 16384
COUNTS = (0, 1, 4095, 4096, 4097, 9024, 16384)


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def voc():
    """ORBvoc's shape (k = 10, L = 6) with leaves at depths 2..6 and 2 % stopped words."""
    return unbalanced_tree(5)


@pytest.fixture(scope="module")
def frames(oracle, voc):
    """The batch: one frame per count in COUNTS plus a frame whose features all land on stopped words and one where 5000 features hit one word."""
    ov = oracle.Vocabulary(voc["k"], voc["L"], voc["parent"], voc["is_leaf"], voc["desc"], voc["weight"])
    out = [frame_features(voc, n, 300 + n) for n in COUNTS]
    rng = np.random.default_rng(301)
    leaves = np.nonzero(voc["is_leaf"])[0]
    stopped_leaves = np.nonzero((voc["is_leaf"] == 1) & (voc["weight"] == 0))[0]
    cand = voc["desc"][rng.choice(stopped_leaves, 20000)] ^ _noise(rng, 20000, 0.01)
    _, _, node, word = ov.transform(cand, 4)
    stopped = cand[(node == -1) & (word >= 0)]
    assert len(stopped) >= 3000
    out.append(stopped[:3000])
    near = voc["desc"][rng.choice(leaves, 100)] ^ _noise(rng, 100, 0.02)
    one = near[np.nonzero(ov.transform(near, 4)[2] >= 0)[0][0]]
    many = np.concatenate([np.repeat(one[None], 5000, axis=0), frame_features(voc, 1000, 302)])
    out.append(many[rng.permutation(len(many))])
    return out


def _batch(frames):
    d = np.full((len(frames), STRIDE, 32), 0xAB, np.uint8)
    for i, f in enumerate(frames):
        d[i, :len(f)] = f
    return d, np.array([len(f) for f in frames], np.int32)


@pytest.mark.parametrize("levelsup", [4, 3, 6])
def test_transform_fv_matches_oracle(oracle, voc, frames, levelsup):
    """levelsup 4 (ComputeBoW's); 3: the depth-2 leaves sit above the FeatureVector level (node 0, the oracle's defined value); 6: node 0 for all."""
    from cubemapslam_b200.vocabulary import Vocabulary
    gv = Vocabulary(voc["k"], voc["L"], voc["parent"], voc["is_leaf"], voc["desc"], voc["weight"], max_frames=len(frames), max_features=64)
    ov = oracle.Vocabulary(voc["k"], voc["L"], voc["parent"], voc["is_leaf"], voc["desc"], voc["weight"])
    d, n = _batch(frames)
    got = gv.transform_fv(d, n=n, levelsup=levelsup)
    dev = _transform_fv_dev(gv, d, n, levelsup)
    for f, feats in enumerate(frames):
        bw, bv, node, _ = ov.transform(feats, levelsup)
        fn, fs, ff = feature_vector(node)
        gbw, gbv, gfn, gfs, gff = got[f]
        assert np.array_equal(gbw, bw) and np.array_equal(gbv.view(np.uint64), bv.view(np.uint64)), "frame %d: BowVector" % f
        assert np.array_equal(gfn, fn) and np.array_equal(gfs, fs) and np.array_equal(gff, ff), "frame %d: FeatureVector" % f
        for a, b in zip(dev[f], got[f]):
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), "frame %d: _dev" % f
    assert len(got[len(COUNTS)][0]) == 0 and len(got[len(COUNTS)][2]) == 0          # every feature stopped: both vectors empty
    big = got[len(COUNTS) + 1]
    assert np.diff(big[3]).max() >= 5000                                            # one node holds the 5000 copies
    if levelsup == 3:
        assert 0 in got[COUNTS.index(16384)][2]                                     # leaves above the FeatureVector level
    gv.close()


def _transform_fv_dev(gv, d, n, levelsup):
    import torch
    from cubemapslam_b200._capi import check, lib, ptr
    F, stride = d.shape[0], d.shape[1]
    dd = torch.from_numpy(d).cuda(); dn = torch.from_numpy(n).cuda()
    i32 = lambda *s: torch.full(s, -7, dtype=torch.int32, device="cuda")
    word, leaf, node, bw, fn, ff = (i32(F, stride) for _ in range(6))
    bv = torch.zeros((F, stride), dtype=torch.float64, device="cuda"); bc, fc = i32(F), i32(F); fs = i32(F, stride + 1)
    torch.cuda.synchronize()
    check(lib().cslam_bow_transform_fv_dev(gv._h, ptr(dd.data_ptr()), ptr(dn.data_ptr()), stride, F, int(levelsup),
                                           *[ptr(t.data_ptr()) for t in (word, leaf, node, bw, bv, bc, fn, fs, ff, fc)]))
    check(lib().cslam_vocabulary_sync(gv._h))
    bw, bv, bc, fn, fs, ff, fc = (t.cpu().numpy() for t in (bw, bv, bc, fn, fs, ff, fc))
    return [(bw[f, :bc[f]], bv[f, :bc[f]], fn[f, :fc[f]], fs[f, :fc[f] + 1], ff[f, :fs[f, fc[f]]]) for f in range(F)]


def test_transform_fv_rejects_stride_past_16384(voc):
    from cubemapslam_b200._capi import CslamError, check, lib, ptr
    from cubemapslam_b200.vocabulary import Vocabulary
    gv = Vocabulary(voc["k"], voc["L"], voc["parent"], voc["is_leaf"], voc["desc"], voc["weight"], max_frames=1, max_features=64)
    with pytest.raises(CslamError, match=r"error -2: cslam_bow_transform_fv: bad argument"):
        gv.transform_fv(np.zeros((STRIDE + 1, 32), np.uint8))
    dummy = np.zeros(1, np.int32)
    with pytest.raises(CslamError, match=r"error -2: cslam_bow_transform_fv_dev: bad argument"):
        check(lib().cslam_bow_transform_fv_dev(gv._h, *[ptr(dummy)] * 2, STRIDE + 1, 1, 4, *[ptr(dummy)] * 10))
    bw, bv, fn, fs, ff = gv.transform_fv(np.zeros((STRIDE, 32), np.uint8))              # the handle still works: one word, or none if stopped
    assert len(bw) == len(fn) <= 1 and fs[-1] == STRIDE * len(fn)
    gv.close()


# ---------------------------------------------------------------------------------------------------- the drop-ins on the reference's objects
@pytest.fixture(scope="module")
def dropin_voc(tmp_path_factory, oracle, voc):
    """libdropin_bow.so with the camera set, and the vocabulary loaded by the reference's loader from a file that ends with a newline."""
    L = dropin_lib()
    L.dropin_set_camera(C.byref(oracle.cam_params(config.lafida_450())))
    path = tmp_path_factory.mktemp("voc") / "voc.txt"
    write_with_newline(voc, path)
    return L, load_vocabulary(L, path)


def _compute(L, h, keyframe, cpu, feats, preset=0):
    n = len(feats); cap = n + 2
    bw = np.zeros(cap, np.int32); bv = np.zeros(cap, np.float64); fn = np.zeros(cap, np.int32); fs = np.zeros(cap + 1, np.int32); ff = np.zeros(cap, np.int32)
    nb = C.c_int32(); nf = C.c_int32()
    d = np.ascontiguousarray(feats, np.uint8).reshape(-1, 32)
    L.dropin_compute_bow(h, int(keyframe), int(cpu), n, _vp(d) if n else None, int(preset), _vp(bw), _vp(bv), C.byref(nb), _vp(fn), _vp(fs), _vp(ff), C.byref(nf))
    j = nf.value
    return bw[:nb.value], bv[:nb.value], fn[:j], fs[:j + 1], ff[:fs[j]]


def _same(a, b):
    return all(x.dtype == y.dtype and np.array_equal(x.view(np.uint8), y.view(np.uint8)) for x, y in zip(a, b))


@pytest.mark.parametrize("keyframe", [0, 1])
@pytest.mark.parametrize("n", [0, 1, 2000, 6024, 9024, 16384])
def test_dropin_compute_bow_equals_reference_body(dropin_voc, voc, keyframe, n):
    """ComputeBoW == ComputeBoW_cpu on identical Frames / KeyFrames; 9024 = a key frame from the initialisation extractor at 3000 features."""
    L, h = dropin_voc
    feats = frame_features(voc, n, 400 + n)
    gpu = _compute(L, h, keyframe, 0, feats)
    cpu = _compute(L, h, keyframe, 1, feats)
    assert _same(gpu, cpu)
    if n == 0:
        assert len(gpu[0]) == 0 and len(gpu[2]) == 0
    else:
        assert len(gpu[0]) > 0 and gpu[3][-1] <= n


def test_dropin_compute_bow_guards(dropin_voc, voc):
    """Frame: an mBowVec already filled is left alone (with its FeatureVector). KeyFrame: mBowVec filled but mFeatVec empty is recomputed;
    both filled is left alone."""
    L, h = dropin_voc
    feats = frame_features(voc, 2000, 500)
    kept = _compute(L, h, 0, 0, feats, preset=1)
    assert list(kept[0]) == [7] and kept[1][0] == 0.5 and len(kept[2]) == 0
    assert _same(kept, _compute(L, h, 0, 1, feats, preset=1))
    fresh = _compute(L, h, 1, 1, feats)
    redone = _compute(L, h, 1, 0, feats, preset=1)
    assert _same(redone, fresh) and _same(_compute(L, h, 1, 1, feats, preset=1), fresh)
    both = _compute(L, h, 1, 0, feats, preset=3)
    assert list(both[0]) == [7] and list(both[2]) == [3] and list(both[4]) == [0]
    assert _same(both, _compute(L, h, 1, 1, feats, preset=3))


def test_dropin_compute_bow_from_concurrent_threads(dropin_voc, voc):
    """Two host threads (a Frame, like Tracking, and a KeyFrame, like LocalMapping) calling ComputeBoW at once, each on its own device handle,
    get the serial results of the reference's bodies; then four."""
    L, h = dropin_voc
    n = 3000
    for nthreads in (2, 4):
        feats = np.stack([frame_features(voc, n, 600 + 10 * nthreads + t) for t in range(nthreads)])
        row = n + 1
        bw = np.zeros((nthreads, row), np.int32); bv = np.zeros((nthreads, row), np.float64); fn = np.zeros((nthreads, row), np.int32)
        fs = np.zeros((nthreads, row), np.int32); ff = np.zeros((nthreads, row), np.int32); nb = np.zeros(nthreads, np.int32); nf = np.zeros(nthreads, np.int32)
        L.dropin_compute_bow_threads(h, nthreads, 5, n, _vp(feats), _vp(bw), _vp(bv), _vp(nb), _vp(fn), _vp(fs), _vp(ff), _vp(nf))
        for t in range(nthreads):
            j = nf[t]
            got = (bw[t, :nb[t]], bv[t, :nb[t]], fn[t, :j], fs[t, :j + 1], ff[t, :fs[t, j]])
            assert _same(got, _compute(L, h, t & 1, 1, feats[t])), "thread %d of %d" % (t, nthreads)
