"""oracle DBoW2 transform (oracle/bow.h) == the reference's own DBoW2 compiled in oracle/_ref/libref.so, on a synthetic vocabulary in ORBvoc.txt's format; the reference's answers are recorded for where
the library cannot be built (tests/refrecord.py)."""
import numpy as np
import pytest

from cubemapslam_b200 import synth

from oracle import ref
from tests.refrecord import RefRecord, same

REC = RefRecord("oracle_bow")


@pytest.mark.parametrize("k,L,levelsup", [(10, 4, 2), (6, 5, 4), (10, 3, 4)])
def test_transform_matches_reference_dbow2(oracle, tmp_path, k, L, levelsup):
    voc = synth.vocabulary(k=k, L=L, seed=k + L)
    ov = oracle.Vocabulary(k, L, voc["parent"], voc["is_leaf"], voc["desc"], voc["weight"])
    rng = np.random.default_rng(1)
    # features near words (realistic) plus pure noise
    leaves = np.nonzero(voc["is_leaf"])[0]
    f1 = voc["desc"][rng.choice(leaves, 1500)] ^ np.packbits(rng.random((1500, 256)) < 0.05, axis=1, bitorder="little")
    feats = np.concatenate([f1, rng.integers(0, 256, (500, 32), dtype=np.uint8)])
    bw, bv, node, word = ov.transform(feats, levelsup)

    def run():
        path = tmp_path / "voc.txt"
        synth.write_vocabulary_text(voc, str(path))
        rv = ref.RefVocabulary(str(path))
        return (rv.size(),) + rv.transform(feats, levelsup)
    size, rbw, rbv, rnode = REC("transform_%d_%d_%d" % (k, L, levelsup), run, digest=(1, 2, 3))
    assert size == k ** L
    assert same(np.asarray(bw, np.int32), rbw) and same(np.asarray(bv, np.float64), rbv)     # BowVector: same words, bit-identical L1-normalised doubles
    assert same(np.asarray(node, np.int32), rnode)                                            # FeatureVector membership of every feature
    assert abs(bv.sum() - 1.0) < 1e-12 and len(bw) > 300
    assert (node[word >= 0] >= 0).mean() > 0.95                           # a few stopped words (weight 0) are excluded like in the reference


def test_transform_unbalanced_tree_with_ties_matches_reference_dbow2(oracle, tmp_path):
    """ORBvoc's shape with 1..10 children per node and leaves at depths 2..6, at levelsup 4 (Frame::ComputeBoW), and features tied between
    two siblings at every level (the first in file order must win): the oracle's descent against the reference's."""
    from tests.test_gpu_bow_limits import unbalanced_features, unbalanced_tree
    voc = unbalanced_tree(0)
    feats, lev, _ = unbalanced_features(voc)
    ov = oracle.Vocabulary(voc["k"], voc["L"], voc["parent"], voc["is_leaf"], voc["desc"], voc["weight"])
    bw, bv, node, word = ov.transform(feats, 4)

    def run():
        path = tmp_path / "voc.txt"
        synth.write_vocabulary_text(voc, str(path))
        rv = ref.RefVocabulary(str(path))
        return (rv.size(),) + rv.transform(feats, 4)
    size, rbw, rbv, rnode = REC("transform_unbalanced_ties", run, digest=(1, 2, 3))
    assert size == int(voc["is_leaf"].sum()) and sorted(set(lev.tolist())) == [1, 2, 3, 4, 5, 6]
    assert same(np.asarray(bw, np.int32), rbw) and same(np.asarray(bv, np.float64), rbv)
    assert same(np.asarray(node, np.int32), rnode)
