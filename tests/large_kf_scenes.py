"""Scenes for the key-frame searches past 4096 features (SearchByBoW in both forms, SearchForTriangulation, Fuse): shared by the oracle-vs-
reference test on the CPU and the GPU tests. Feature counts are those of the initialisation extractor's key frames (3*nFeatures + 3*nlevels:
6024 at 2000 features, 9024 at 3000) and the seams around 4096."""
import numpy as np

from cubemapslam_b200 import synth
from oracle.oracle import KP_DTYPE

SIZES = (4097, 6024, 9024)


def bow_pair(n1, n2, seed):
    """Two sides of a SearchByBoW call: side 2 holds noisy copies of side 1's descriptors in the same FeatureVector node, ~6 features per node,
    5 % of each side in no node (node -1). Where the indices exist, side-2 features a, a + 4096 and a + 8192 of some anchors a are identical
    copies in one node (ties 4096 and 8192 apart), and side-1 features b and b + 4096 too (the second must skip what the first took)."""
    rng = np.random.default_rng(7000 + seed)
    nn = max(1, max(n1, n2) // 6)
    d1 = rng.integers(0, 256, (n1, 32), dtype=np.uint8); node1 = rng.integers(0, nn, n1).astype(np.int32)
    src = rng.integers(0, max(n1, 1), n2) if n1 else np.zeros(n2, np.int64)
    d2 = rng.integers(0, 256, (n2, 32), dtype=np.uint8); node2 = rng.integers(0, nn, n2).astype(np.int32)
    if n1:
        copy = rng.random(n2) < 0.75
        flips = np.packbits(rng.random((n2, 256)) < 0.04, axis=1, bitorder="little")
        d2[copy] = d1[src[copy]] ^ flips[copy]; node2[copy] = node1[src[copy]]
    for a in range(0, n2, 97):
        for k in (4096, 8192):
            if a + k < n2:
                d2[a + k] = d2[a]; node2[a + k] = node2[a]
    for b in range(0, n1, 89):
        if b + 4096 < n1:
            d1[b + 4096] = d1[b]; node1[b + 4096] = node1[b]
    node1[rng.random(n1) < 0.05] = -1; node2[rng.random(n2) < 0.05] = -1
    a1 = rng.uniform(0, 360, n1).astype(np.float32)
    a2 = np.mod(a1[np.minimum(src, max(n1 - 1, 0))] + rng.uniform(-8, 8, n2).astype(np.float32), np.float32(360)).astype(np.float32) if n1 else \
        rng.uniform(0, 360, n2).astype(np.float32)
    a2[a2 >= 360] = 0
    v1 = (rng.random(n1) < 0.85).astype(np.uint8); v2 = (rng.random(n2) < 0.85).astype(np.uint8)
    return dict(d1=d1, a1=a1, v1=v1, node1=node1, d2=d2, a2=a2, v2=v2, node2=node2)


def key_points(ang):
    k = np.zeros(len(ang), KP_DTYPE); k["x"] = 600; k["y"] = 600; k["angle"] = ang
    return k


def oracle_nodes(node, side):
    """Per-feature node ids for the oracle, whose FeatureVector groups every id: features in no node get an id of their own side only."""
    return np.where(node < 0, -2 - side, node).astype(np.int32)


def csr(node, stride):
    """The FeatureVector of per-feature node ids (-1: in no node) in cslam_bow_transform_fv's layout: (node, start, feat)."""
    idx = np.nonzero(node >= 0)[0]
    order = idx[np.argsort(node[idx], kind="stable")]
    nodes, first = np.unique(node[order], return_index=True)
    start = np.append(first, len(order)).astype(np.int32)
    assert len(nodes) <= stride
    return nodes.astype(np.int32), start, order.astype(np.int32)


def mapping_pair(n, seed):
    """synth.mapping_pair (face width 650) with exactly n key points on both key frames: generated larger, then both cut to n (the current
    frame's count varies around the requested one)."""
    s = synth.mapping_pair(seed, n=n + n // 8 + 8, faceW=650)
    assert len(s["kCur"]) >= n and len(s["kLast"]) >= n
    for k in ("kCur", "dCur", "hasMPCur", "nodeCur", "src"):
        s[k] = np.ascontiguousarray(s[k][:n])
    for k in ("kLast", "dLast", "hasMPObs", "nodeObs", "Xw"):
        s[k] = np.ascontiguousarray(s[k][:n])
    return s
