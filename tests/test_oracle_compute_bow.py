"""The vocabulary import of dropin/ComputeBoW_b200.cpp (Frame::ComputeBoW / KeyFrame::ComputeBoW on the GPU) copies the reference's loaded
ORBVocabulary object, not ORBvoc.txt: its arrays, fed to the oracle (oracle/bow.h), must reproduce the reference's own DBoW2 transform on that
object bit for bit - BowVector words and double bits, FeatureVector nodes and index lists - at 0, 1, 2000, 6024 and 9024 features (9024 = an
initialisation key frame at 3000 features). Vocabularies: synthetic ones written with and without the trailing newline that ORBvoc.txt ends
with (the loader's while(!f.eof()) loop makes one more node of it), and ORBvoc.txt itself. The importer runs in oracle/_ref/libdropin_bow.so
without touching the GPU; the reference's answers are recorded (tests/refrecord.py)."""
import ctypes as C
import os
import tarfile

import numpy as np
import pytest

from cubemapslam_b200 import synth
from oracle import ref
from tests.refrecord import RefRecord, same
from tests.test_gpu_bow_limits import _noise, unbalanced_tree

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DROPIN = os.path.join(ROOT, "oracle", "_ref", "libdropin_bow.so")
REF = os.environ.get("REF", "/root/reference")
ORBVOC = os.path.join(REF, "Vocabulary", "ORBvoc.txt.tar.gz")
COUNTS = (0, 1, 2000, 6024, 9024)
REC = RefRecord("oracle_compute_bow")


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def dropin_lib():
    if not os.path.exists(DROPIN):
        pytest.skip("oracle/_ref/libdropin_bow.so is built where the reference tree exists")
    return C.CDLL(DROPIN)


def load_vocabulary(L, path):
    """ORBVocabulary::loadFromTextFile in libdropin_bow.so; the object's address."""
    h = C.c_void_p()
    assert L.dropin_voc_load(str(path).encode(), C.byref(h)) == 0 and h.value, path
    return h


class LoadedVocabulary:
    """An ORBVocabulary loaded by the reference's loadFromTextFile inside libdropin_bow.so, and the drop-in importer's arrays of it. It is never
    freed: the drop-in imports a vocabulary once per address, for a process-long object like System's."""

    def __init__(self, L, path):
        self.L = L
        self.h = load_vocabulary(L, path)
        info = np.zeros(4, np.int32)
        L.dropin_voc_info(self.h, _vp(info))
        self.k, self.L_levels, n, self.size = (int(x) for x in info)
        self.parent = np.zeros(n, np.int32); self.is_leaf = np.zeros(n, np.uint8); self.desc = np.zeros((n, 32), np.uint8); self.weight = np.zeros(n, np.float64)
        L.dropin_voc_export(self.h, _vp(self.parent), _vp(self.is_leaf), _vp(self.desc), _vp(self.weight))

    def arrays(self):
        return dict(k=self.k, L=self.L_levels, parent=self.parent, is_leaf=self.is_leaf, desc=self.desc, weight=self.weight)


def write_with_newline(voc, path):
    """synth.write_vocabulary_text, then the final newline ORBvoc.txt has."""
    synth.write_vocabulary_text(voc, str(path))
    with open(path, "a") as f:
        f.write("\n")


def frame_features(voc, n, seed):
    """n descriptors: 85 % near a word (5 % of the bits flipped), the rest uniform noise."""
    rng = np.random.default_rng(seed)
    leaves = np.nonzero(voc["is_leaf"])[0]
    near = int(0.85 * n)
    f = voc["desc"][rng.choice(leaves, near)] ^ _noise(rng, near, 0.05)
    return np.concatenate([f, rng.integers(0, 256, (n - near, 32), dtype=np.uint8)]).astype(np.uint8)


def feature_vector(node):
    """FeatureVector (std::map<NodeId, std::vector<unsigned>>) from per-feature nodes (-1: in none) as CSR: nodes, starts, feature indices."""
    live = np.nonzero(node >= 0)[0]
    order = live[np.argsort(node[live], kind="stable")]
    nodes, first = np.unique(node[order], return_index=True)
    return nodes.astype(np.int32), np.append(first, len(order)).astype(np.int32), order.astype(np.int32)


def _check(oracle, key, voc_arrays, path, feats_of):
    ov = oracle.Vocabulary(voc_arrays["k"], voc_arrays["L"], voc_arrays["parent"], voc_arrays["is_leaf"], voc_arrays["desc"], voc_arrays["weight"])
    rv = []

    def reference():
        if not rv:
            rv.append(ref.RefVocabulary(str(path())))
        return rv[0]
    for n in COUNTS:
        feats = feats_of(n)
        bw, bv, node, _ = ov.transform(feats, 4)
        rbw, rbv, rnode = REC("%s_%d" % (key, n), lambda: reference().transform(feats, 4), digest=(0, 1, 2))
        assert same(np.asarray(bw, np.int32), rbw) and same(np.asarray(bv, np.float64), rbv), "%s, %d features: BowVector" % (key, n)
        assert same(np.asarray(node, np.int32), rnode), "%s, %d features: FeatureVector" % (key, n)
        fn, fs, ff = feature_vector(node)
        assert len(bw) <= n and fs[-1] == (node >= 0).sum() and (n == 0 or len(fn) > 0)


@pytest.mark.parametrize("newline", [False, True])
def test_imported_synthetic_vocabulary_reproduces_reference(oracle, tmp_path, newline):
    L = dropin_lib()
    voc = unbalanced_tree(3)
    path = tmp_path / "voc.txt"
    (write_with_newline if newline else synth.write_vocabulary_text)(voc, path)
    lv = LoadedVocabulary(L, path)
    n = len(voc["parent"])
    assert same(lv.parent[:n], voc["parent"]) and same(lv.is_leaf[:n], voc["is_leaf"]) and same(lv.desc[:n], voc["desc"]) and same(lv.weight[:n], voc["weight"])
    if newline:   # the empty last line: one more word, stopped (weight 0), in the children of the last line's parent
        assert len(lv.parent) == n + 1 and lv.size == int(voc["is_leaf"].sum()) + 1
        assert lv.parent[n] == voc["parent"][-1] and lv.is_leaf[n] == 1 and lv.weight[n] == 0.0
    else:
        assert len(lv.parent) == n and lv.size == int(voc["is_leaf"].sum())
    arrays = lv.arrays()
    _check(oracle, "synthetic_%s" % ("newline" if newline else "plain"), arrays, lambda: path, lambda c: frame_features(voc, c, 100 + c))


def test_imported_orbvoc_reproduces_reference(oracle, tmp_path):
    """ORBvoc.txt as shipped: 1 082 073 nodes once loaded, 971 815 words where the file lists 971 814 leaves."""
    L = dropin_lib()
    if not os.path.exists(ORBVOC):
        pytest.skip("ORBvoc.txt comes from the reference tree")
    with tarfile.open(ORBVOC) as t:
        t.extractall(tmp_path, filter="data")
    path = tmp_path / "ORBvoc.txt"
    lv = LoadedVocabulary(L, path)
    assert (lv.k, lv.L_levels, len(lv.parent), lv.size) == (10, 6, 1082073, 971815)
    assert int(lv.is_leaf[:-1].sum()) == 971814
    assert lv.parent[-1] == lv.parent[-2] and lv.is_leaf[-1] == 1 and lv.weight[-1] == 0.0
    depth = np.zeros(len(lv.parent) + 1, np.int64)
    for _ in range(6):
        depth[1:] = depth[lv.parent] + 1
    words = np.nonzero(lv.is_leaf)[0] + 1
    assert int((depth[words] < 6).sum()) == 820
    arrays = lv.arrays()
    # features from the file's own words: the extra node's descriptor bytes are whatever memory FORB::fromString left (zero here)
    listed = dict(is_leaf=arrays["is_leaf"][:-1], desc=arrays["desc"][:-1])
    _check(oracle, "orbvoc", arrays, lambda: path, lambda c: frame_features(listed, c, 200 + c))
