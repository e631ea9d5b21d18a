"""The three kernels that rebuild DBoW2 structures from packed sort keys `id << 12 | feature index` (k_bow_vector: word, k_search_by_bow:
FeatureVector node, k_triangulation: KF2's node) at the top of both key fields: feature indices 2048..4095 (every key frame of the 3000-feature
camera configurations lives there) and ids up to 2^20 - 2 (ORBvoc.txt has ~10^6 words), with ties built on purpose for each kernel's
first- / last-minimum rule, node -1 (a stopped word's feature, in no FeatureVector node) and the host-side node-id range checks.
Every answer is compared with the oracle, exactly; the oracle's transform is pinned to the compiled reference DBoW2 in tests/test_oracle_bow.py."""
import numpy as np
import pytest

from cubemapslam_b200 import synth

pytestmark = pytest.mark.gpu

STRIDE = 4096
ID_END = (1 << 20) - 1                     # node / word ids the keys hold apart: [-1, 2^20 - 1)
BOW_SENTINELS = (0x7ffff, 0x7fffe)         # ORBMatcher_b200.cpp: KF / F features in no FeatureVector node
TRI_SENTINELS = ((1 << 20) - 3, (1 << 20) - 2)   # ORBMatcher_mapping_b200.cpp: KF1 / KF2 likewise
POPC = np.array([bin(i).count("1") for i in range(256)], np.int32)


# ----------------------------------------------------------------------------------------------------------------- generators
def _flip_mask(rng, shape):
    """Random bit mask with ~12.5 % of the bits set (AND of three uniform byte arrays)."""
    return rng.integers(0, 256, shape, dtype=np.uint8) & rng.integers(0, 256, shape, dtype=np.uint8) & rng.integers(0, 256, shape, dtype=np.uint8)


def _noise(rng, n, p):
    return np.packbits(rng.random((n, 256)) < p, axis=1, bitorder="little")


def balanced_tree(k, L, seed, stop_frac=0.05, drop_last_leaves=0):
    """Vocabulary tree in ORBvoc.txt's breadth-first node order (children of one parent consecutive, parents in file order), built level by
    level: a child is its parent with ~12 % of the bits flipped. The last `drop_last_leaves` leaves are left out (the file's last lines)."""
    rng = np.random.default_rng(seed)
    parents, descs = [], []
    prev_ids = np.zeros(1, np.int64); prev_desc = rng.integers(0, 256, (1, 32), dtype=np.uint8); next_id = 1
    for _ in range(L):
        n = len(prev_ids) * k
        parents.append(np.repeat(prev_ids, k))
        d = np.repeat(prev_desc, k, axis=0) ^ _flip_mask(rng, (n, 32))
        descs.append(d)
        prev_ids = np.arange(next_id, next_id + n, dtype=np.int64); prev_desc = d; next_id += n
    parent = np.concatenate(parents).astype(np.int32); desc = np.concatenate(descs)
    nleaf = k ** L
    is_leaf = np.zeros(len(parent), np.uint8); is_leaf[-nleaf:] = 1
    weight = np.zeros(len(parent), np.float64)
    w = rng.uniform(0.5, 9.0, nleaf); w[rng.random(nleaf) < stop_frac] = 0.0
    weight[-nleaf:] = w
    n = len(parent) - drop_last_leaves
    return dict(k=k, L=L, parent=parent[:n], is_leaf=is_leaf[:n], desc=desc[:n], weight=weight[:n])


def unbalanced_tree(seed=0, k=10, L=6, leaf_prob=0.3):
    """ORBvoc's shape (k = 10, L = 6) with 1..k children per internal node and leaves at depths 2..L (never above depth 2: at levelsup 4 the
    FeatureVector node sits at depth 2, and the reference leaves it unwritten for a shallower leaf). Breadth-first file order, built per level."""
    rng = np.random.default_rng(7100 + seed)
    parents, descs, leaves = [], [], []
    prev_ids = np.zeros(1, np.int64); prev_desc = rng.integers(0, 256, (1, 32), dtype=np.uint8); next_id = 1
    for level in range(1, L + 1):
        cnt = np.full(len(prev_ids), k) if level == 1 else rng.integers(1, k + 1, len(prev_ids))
        n = int(cnt.sum())
        parents.append(np.repeat(prev_ids, cnt))
        d = np.repeat(prev_desc, cnt, axis=0) ^ _flip_mask(rng, (n, 32))
        leaf = np.ones(n, bool) if level == L else (rng.random(n) < leaf_prob) & (level >= 2)
        descs.append(d); leaves.append(leaf)
        ids = np.arange(next_id, next_id + n, dtype=np.int64); next_id += n
        prev_ids, prev_desc = ids[~leaf], d[~leaf]
    parent = np.concatenate(parents).astype(np.int32); is_leaf = np.concatenate(leaves).astype(np.uint8); desc = np.concatenate(descs)
    weight = np.where(is_leaf == 1, rng.uniform(0.5, 9.0, len(parent)), 0.0)
    weight[(is_leaf == 1) & (rng.random(len(parent)) < 0.02)] = 0.0
    return dict(k=k, L=L, parent=parent, is_leaf=is_leaf, desc=desc, weight=weight)


class _Tree:
    """numpy view of a vocabulary for building and checking test features: children lists, depths, word -> leaf node."""

    def __init__(self, voc):
        self.voc = voc
        par = voc["parent"]; N = len(par) + 1
        self.par = np.concatenate([[-1], par]).astype(np.int64)
        self.desc = np.concatenate([np.zeros((1, 32), np.uint8), voc["desc"]])
        self.leaf = np.concatenate([[0], voc["is_leaf"]]).astype(bool)
        self.start = np.searchsorted(par, np.arange(N + 1), side="left") + 1    # children of p: node ids start[p] .. start[p+1]-1 (file order)
        self.depth = np.zeros(N, np.int64)
        for _ in range(voc["L"]):                                                # parents precede children: L sweeps settle every depth
            self.depth[1:] = self.depth[self.par[1:]] + 1
        self.word_leaf = np.nonzero(self.leaf)[0]                                # word id -> leaf node id

    def children(self, p):
        return np.arange(self.start[p], self.start[p + 1])

    def dist(self, f, ids):
        return POPC[self.desc[ids] ^ f].sum(axis=1)

    def descend(self, f):
        """DBoW2's greedy descent, first minimum in file order. Returns [(node, children, distances), ...] per level."""
        path, node = [], 0
        while not self.leaf[node]:
            c = self.children(node); d = self.dist(f, c)
            path.append((int(c[int(np.argmin(d))]), c, d)); node = path[-1][0]
        return path

    def descend_balanced(self, feats, k):
        """The same descent for many features of a balanced tree (at most k children, leaves all at depth L): leaf node id per feature."""
        node = np.zeros(len(feats), np.int64)
        while not self.leaf[node[0]]:
            c = np.minimum(self.start[node][:, None] + np.arange(k), self.start[node + 1][:, None] - 1)   # a short list repeats its last child
            d = POPC[self.desc[c] ^ feats[:, None, :]].sum(axis=2)
            node = c[np.arange(len(feats)), np.argmin(d, axis=1)]
        return node

    def ancestor(self, node, depth):
        while self.depth[node] > depth:
            node = self.par[node]
        return int(node)


def tie_features(voc, seed=0, per_kind=6):
    """Features at equal Hamming distance from two siblings a < b (file order) at one level of their descent, the tie being the minimum
    over all siblings: a's descriptor with half of the bits in which a and b differ (an even number) copied from b. For every level
    1..L, pairs of adjacent siblings and of the first and last sibling. Returns (features, level, a) per feature."""
    T = _Tree(voc); rng = np.random.default_rng(7200 + seed)
    internal = np.nonzero(~T.leaf)[0]
    feats, lev, first = [], [], []
    for level in range(1, voc["L"] + 1):
        cands = internal[(T.depth[internal] == level - 1) & (T.start[internal + 1] - T.start[internal] >= 2)]
        for far in (False, True):
            got = 0
            for _ in range(4000):
                if got == per_kind or len(cands) == 0:
                    break
                c = T.children(int(rng.choice(cands)))
                i = 0 if far else int(rng.integers(0, len(c) - 1))
                a, b = int(c[i]), int(c[-1] if far else c[i + 1])
                diff = np.unpackbits(T.desc[a] ^ T.desc[b], bitorder="little")
                pos = np.nonzero(diff)[0]
                if len(pos) == 0 or len(pos) % 2:
                    continue
                bits = np.unpackbits(T.desc[a], bitorder="little")
                take = rng.choice(pos, len(pos) // 2, replace=False)
                bits[take] ^= 1
                f = np.packbits(bits, bitorder="little")
                path = T.descend(f)
                step = path[level - 1] if len(path) >= level else None
                if step is None or a not in step[1] or b not in step[1]:
                    continue                                      # the descent left a's parent before this level
                d = dict(zip(step[1].tolist(), step[2].tolist()))
                if d[a] != d[b] or d[a] != min(d.values()) or step[0] != a:
                    continue
                feats.append(f); lev.append(level); first.append(a); got += 1
    return np.stack(feats), np.array(lev), np.array(first)


def unbalanced_features(voc, seed=0):
    """The features of the unbalanced-tree case: tie features, features near leaves and pure noise."""
    rng = np.random.default_rng(7300 + seed)
    tf, lev, first = tie_features(voc, seed)
    leaves = np.nonzero(voc["is_leaf"])[0]
    near = voc["desc"][rng.choice(leaves, 900)] ^ _noise(rng, 900, 0.04)
    noise = rng.integers(0, 256, (150, 32), dtype=np.uint8)
    return np.concatenate([tf, near, noise]), lev, first


def _frames_to_stride(frames, stride=STRIDE):
    d = np.full((len(frames), stride, 32), 0xAB, np.uint8)
    for i, f in enumerate(frames):
        d[i, :min(len(f), stride)] = f[:stride]
    return d


def _voc_pair(voc, max_frames, max_features=STRIDE):
    from cubemapslam_b200.vocabulary import Vocabulary
    import oracle as orc
    args = (voc["k"], voc["L"], voc["parent"], voc["is_leaf"], voc["desc"], voc["weight"])
    return Vocabulary(*args, max_frames=max_frames, max_features=max_features), orc.Vocabulary(*args)


def _transform_dev(gv, d, n, levelsup):
    """cslam_bow_transform_dev on device copies of (F, stride, 32) descriptors; returns host word, leaf, node, bow_word, bow_val, bow_count."""
    import torch
    from cubemapslam_b200._capi import check, lib, ptr
    F, stride = d.shape[0], d.shape[1]
    dd = torch.from_numpy(d).cuda(); dn = torch.from_numpy(np.ascontiguousarray(n, np.int32)).cuda()
    out = [torch.full((F, stride), -7, dtype=torch.int32, device="cuda") for _ in range(4)]
    bv = torch.zeros((F, stride), dtype=torch.float64, device="cuda"); bc = torch.zeros(F, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    check(lib().cslam_bow_transform_dev(gv._h, *[ptr(t.data_ptr()) for t in (dd, dn)], stride, F, int(levelsup),
                                        *[ptr(t.data_ptr()) for t in (*out, bv, bc)]))
    check(lib().cslam_vocabulary_sync(gv._h))
    return [t.cpu().numpy() for t in out] + [bv.cpu().numpy(), bc.cpu().numpy()]


# ----------------------------------------------------------------------------------------------------------------- 1. BoW transform at 2^20 - 1 words
K_BIG, L_BIG = 16, 5                        # 16^5 = 2^20 leaves; the tree below drops the last one


@pytest.fixture(scope="module")
def big_tree():
    voc = balanced_tree(K_BIG, L_BIG, seed=1, stop_frac=0.05, drop_last_leaves=1)
    voc["weight"][-1] = 3.0                 # the last word, 2^20 - 2, is not stopped: its keys reach the top of the word field
    return voc


@pytest.fixture(scope="module")
def big_frames(big_tree):
    """Eight frames at stride 4096 (counts 4096, 4095, 3000, 2049, 1, 0, 5000 and one frame of stopped words only), rows past each count 0xAB."""
    voc = big_tree; rng = np.random.default_rng(31)
    T = _Tree(voc); W = len(T.word_leaf); leaf_desc = T.desc[T.word_leaf]
    top = np.arange(int(0.99 * W), W)
    counts = [4096, 4095, 3000, 2049, 1, 0, 5000, 4096]
    frames = []
    for f, c in enumerate(counts[:7]):
        m = min(c, STRIDE)
        words = np.where(rng.random(m) < 0.9, rng.choice(top, m), rng.integers(0, W, m))
        if m > 2048:                        # repeated words on both sides of index 2048
            j = rng.choice(m - 2048, min(200, m - 2048), replace=False)
            words[2048 + j] = words[j]
        x = leaf_desc[words] ^ _noise(rng, m, 0.02)
        if m == STRIDE:
            x[STRIDE - 1] = leaf_desc[W - 1]   # key (2^20 - 2) << 12 | 4095
        frames.append(x)
    stopped = np.nonzero(voc["weight"][voc["is_leaf"] == 1] == 0)[0]
    cand = leaf_desc[rng.choice(stopped, 2 * STRIDE)]
    lands = voc["weight"][T.descend_balanced(cand, K_BIG) - 1] == 0          # keep the ones whose descent ends on a stopped word
    frames.append(cand[lands][:STRIDE])
    assert len(frames[-1]) == STRIDE
    return frames, np.array(counts, np.int32)


def test_vocabulary_word_limit(big_tree):
    from cubemapslam_b200._capi import CslamError
    from cubemapslam_b200.vocabulary import Vocabulary
    full = balanced_tree(K_BIG, L_BIG, seed=1, stop_frac=0.05)
    assert int(full["is_leaf"].sum()) == 1 << 20 and int(big_tree["is_leaf"].sum()) == (1 << 20) - 1
    with pytest.raises(CslamError, match=r"error -2: vocabulary has 1048576 words"):
        Vocabulary(K_BIG, L_BIG, full["parent"], full["is_leaf"], full["desc"], full["weight"], max_frames=1, max_features=64)
    v = Vocabulary(K_BIG, L_BIG, big_tree["parent"], big_tree["is_leaf"], big_tree["desc"], big_tree["weight"], max_frames=1, max_features=64)
    v.close()


@pytest.mark.parametrize("levelsup", [0, 2, 4, L_BIG, L_BIG + 1])
def test_bow_transform_at_top_of_key_fields(big_tree, big_frames, levelsup):
    frames, counts = big_frames
    gv, ov = _voc_pair(big_tree, max_frames=len(frames))
    d = _frames_to_stride(frames)
    host = gv.transform(d, n=counts, levelsup=levelsup)
    word_d, leaf_d, node_d, bw_d, bv_d, bc_d = _transform_dev(gv, d, counts, levelsup)
    T = _Tree(big_tree)
    wid = np.full(len(T.par), -1, np.int64); wid[T.word_leaf] = np.arange(len(T.word_leaf))
    top_key = 0
    for f in range(len(frames)):
        m = min(int(counts[f]), STRIDE)
        bw, bv, node, word = ov.transform(d[f, :m], levelsup)
        gw, gn, gbw, gbv = host[f]
        assert np.array_equal(gw, word) and np.array_equal(gn, node), "frame %d: word / node" % f
        assert np.array_equal(gbw, bw) and np.array_equal(gbv.view(np.uint64), bv.view(np.uint64)), "frame %d: BowVector" % f
        assert bc_d[f] == len(bw) and np.array_equal(bw_d[f, :len(bw)], bw) and np.array_equal(bv_d[f, :len(bw)].view(np.uint64), bv.view(np.uint64))
        assert np.array_equal(word_d[f, :m], word) and np.array_equal(node_d[f, :m], node) and np.array_equal(wid[leaf_d[f, :m]], word)
        assert np.all(np.isfinite(gbv))
        live = node >= 0
        if live.any():
            top_key = max(top_key, int(((word[live].astype(np.int64) << 12) | np.nonzero(live)[0]).max()))
        if m > 2048 and f < 7:              # one word with features on both sides of index 2048
            lo, hi = set(word[:2048][live[:2048]].tolist()), set(word[2048:][live[2048:]].tolist())
            assert lo & hi, "frame %d" % f
    assert top_key == ((1 << 20) - 2) << 12 | 4095
    assert len(host[7][2]) == 0 and np.all(host[7][1] == -1)            # every feature on a stopped word: empty BowVector, no NaN
    assert len(host[5][0]) == 0 and len(host[4][0]) == 1 and len(host[6][0]) == STRIDE
    stopped = sum(int((h[1] == -1).sum()) for h in host[:7]); total = sum(len(h[1]) for h in host[:7])
    assert 0.02 < stopped / total < 0.1
    gv.close()


# ----------------------------------------------------------------------------------------------------------------- 2. unbalanced tree, ties
def test_bow_transform_unbalanced_tree_ties():
    voc = unbalanced_tree(0)
    T = _Tree(voc)
    depths = T.depth[T.word_leaf]
    assert depths.min() == 2 and depths.max() == 6 and len(set(depths.tolist())) == 5
    feats, lev, first = unbalanced_features(voc)
    assert sorted(set(lev.tolist())) == [1, 2, 3, 4, 5, 6]
    gv, ov = _voc_pair(voc, max_frames=1)
    bw, bv, node, word = ov.transform(feats, 4)
    gw, gn, gbw, gbv = gv.transform(feats, levelsup=4)
    assert np.array_equal(gw, word) and np.array_equal(gn, node)
    assert np.array_equal(gbw, bw) and np.array_equal(gbv.view(np.uint64), bv.view(np.uint64))
    word_d, leaf_d, node_d, *_ = _transform_dev(gv, feats[None], [len(feats)], 4)
    assert np.array_equal(leaf_d[0, :len(feats)], T.word_leaf[word])
    for i in range(len(lev)):                # the first sibling in file order wins every tie
        assert T.ancestor(int(T.word_leaf[gw[i]]), lev[i]) == first[i], "tie feature %d at level %d" % (i, lev[i])
    gv.close()


# ----------------------------------------------------------------------------------------------------------------- 3. SearchByBoW at 4096
BIG_NODE = 7


def bow_pair(seed, nKF, nF):
    """A (KF, F) pair for SearchByBoW with node ids that reach the top of the id field and ties by construction. F rows are noisy copies
    of KF rows (or fresh). Nodes: level-2 ids, the drop-in sentinels on both sides, 2^20 - 2 on both sides, one node of > 1024 features on
    both sides where both are large, many one-feature nodes. Duplicate F descriptors in the big node at group positions p and p + 32 m
    (one lane) and p, p + 7 (two lanes), on both sides of index 2048, each with one KF query near it."""
    rng = np.random.default_rng(7400 + seed)
    dK = rng.integers(0, 256, (nKF, 32), dtype=np.uint8); aK = rng.uniform(0, 360, nKF).astype(np.float32)
    src = rng.integers(0, nKF, nF); fresh = rng.random(nF) < 0.2
    dF = dK[src] ^ _noise(rng, nF, 0.05); dF[fresh] = rng.integers(0, 256, (int(fresh.sum()), 32), dtype=np.uint8)
    aF = np.mod(aK[src] + rng.uniform(-5, 5, nF), 360).astype(np.float32); aF[aF >= 360] = 0
    pool = np.array(list(range(11, 111)) + list(BOW_SENTINELS) + [ID_END - 1], np.int32)
    nK = rng.choice(pool, nKF).astype(np.int32)
    single = rng.random(nKF) < 0.08
    nK[single] = 200000 + np.nonzero(single)[0]                       # one-feature nodes (the F copy joins it)
    big = min(nKF, nF) >= 3000
    if big:
        nK[rng.choice(nKF, 1500, replace=False)] = BIG_NODE
    nFd = nK[src].copy()
    re = rng.random(nF) < 0.1
    nFd[re] = rng.choice(pool, int(re.sum()))
    valid = (rng.random(nKF) < 0.85).astype(np.uint8)
    if big:
        G = np.nonzero(nFd == BIG_NODE)[0]                              # the big node's F list (ascending index = list order)
        assert len(G) > 1024 and (nK == BIG_NODE).sum() > 1024
        r0 = int(np.searchsorted(G, 2048))
        pairs = [(r0 - 40, r0 - 40 + 32), (r0 - 100, r0 - 100 + 96), (r0 - 3, r0 + 4), (r0 + 20, r0 + 20 + 64), (r0 + 50, r0 + 57), (10, 11), (30, 30 + 32 * 5)]
        qs = rng.choice(np.nonzero(nK == BIG_NODE)[0], len(pairs), replace=False)
        for (p1, p2), q in zip(pairs, qs):
            D = rng.integers(0, 256, 32, dtype=np.uint8)
            dF[G[p1]] = D; dF[G[p2]] = D
            aF[G[p1]] = aF[G[p2]] = aK[q]
            dK[q] = D ^ _noise(rng, 1, 0.04)[0]; valid[q] = 1
    return dK, aK, valid, nK, dF, aF, nFd


def _batch(pairs):
    return [np.stack([p[i] for p in pairs]) for i in range(7)]


def _search_dev(m, a):
    import torch
    P, nKF, nF = a[0].shape[0], a[0].shape[1], a[4].shape[1]
    t = [torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in a]
    mf = torch.full((P, nF), -7, dtype=torch.int32, device="cuda"); nm = torch.zeros(P, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    m.search_by_bow_dev(t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(), nKF, t[4].data_ptr(), t[5].data_ptr(), t[6].data_ptr(), nF, P,
                        mf.data_ptr(), nm.data_ptr())
    m.sync()
    return nm.cpu().numpy(), mf.cpu().numpy()


@pytest.fixture(scope="module")
def matcher4096():
    from cubemapslam_b200.matcher import ORBMatcher
    m = ORBMatcher(0.7, True, max_pairs=3, max_features=STRIDE)
    yield m
    m.close()


@pytest.mark.parametrize("nKF,nF", [(4096, 4096), (4096, 1), (1, 4096), (4096, 2049), (3000, 3000)])
def test_search_by_bow_at_4096(oracle, matcher4096, nKF, nF):
    m = matcher4096
    pairs = [bow_pair(10 * nKF + nF + p, nKF, nF) for p in range(3)]
    a = _batch(pairs)
    valid2 = np.stack([(np.random.default_rng(p).random(nF) < 0.85).astype(np.uint8) for p in range(3)])
    hiK = hiF = 0
    # nnratio 0.7: equal best and second best are rejected; 1.5: they pass, and the earliest list position must win
    for nnratio in (0.7, 1.5):
        m.nnratio = nnratio
        nm, mf = m.SearchByBoW(*a)
        dn, dmf = _search_dev(m, a)
        kn, k12 = m.SearchByBoW_KF(a[0], a[1], a[2], a[3], a[4], a[5], valid2, a[6])
        for p in range(3):
            rn, rm = oracle.search_by_bow(*[x[p] for x in a], nnratio, True)
            assert nm[p] == rn and np.array_equal(mf[p], rm), "pair %d, nnratio %g" % (p, nnratio)
            assert dn[p] == rn and np.array_equal(dmf[p], rm), "pair %d, nnratio %g (_dev)" % (p, nnratio)
            r2n, r12 = oracle.search_by_bow_kf(a[0][p], a[1][p], a[2][p], a[3][p], a[4][p], a[5][p], valid2[p], a[6][p], nnratio, True)
            assert kn[p] == r2n and np.array_equal(k12[p], r12), "pair %d, nnratio %g (KeyFrame overload)" % (p, nnratio)
            hit = rm >= 0
            if hit.any():
                hiK = max(hiK, int(rm[hit].max())); hiF = max(hiF, int(np.nonzero(hit)[0].max()))
            if min(nKF, nF) >= 3000:
                assert rn > 300
                nK, nFd = a[3][p], a[6][p]
                for s in (*BOW_SENTINELS, ID_END - 1, BIG_NODE):    # matches in the top and the largest node ids
                    assert np.any(hit & (nFd == s) & (nK[np.maximum(rm, 0)] == s)), "no match in node %d" % s
    if min(nKF, nF) >= 3000:
        assert hiK >= 2048 and hiF >= 2048
    m.nnratio = 0.7


def test_search_by_bow_ties(oracle, matcher4096):
    """The tie rows of bow_pair on their own terms: at nnratio 0.7 no duplicate wins, at 1.5 every duplicate pair is matched at its earlier row."""
    m = matcher4096
    a = _batch([bow_pair(1, 4096, 4096)])
    G = np.nonzero(a[6][0] == BIG_NODE)[0]
    seen, dup = {}, []
    for i in G:
        key = a[4][0, i].tobytes()
        if key in seen:
            dup.append((seen[key], int(i)))
        seen[key] = int(i)
    assert len(dup) == 7 and any(i < 2048 <= j for i, j in dup) and any(i >= 2048 for i, j in dup)
    lanes = [(np.searchsorted(G, j) - np.searchsorted(G, i)) % 32 for i, j in dup]   # list positions p, p + 32 m share a lane
    assert 0 in lanes and any(lanes)
    for nnratio in (0.7, 1.5):
        m.nnratio = nnratio
        nm, mf = m.SearchByBoW(*a)
        rn, rm = oracle.search_by_bow(*[x[0] for x in a], nnratio, True)
        assert nm[0] == rn and np.array_equal(mf[0], rm)
        for i, j in dup:
            assert mf[0, j] == -1 and (mf[0, i] == -1) == (nnratio < 1)
    m.nnratio = 0.7


@pytest.mark.parametrize("bad", [ID_END, 1 << 20, (1 << 20) + 5, -2])
def test_search_by_bow_rejects_node_ids_outside_range(matcher4096, bad):
    from cubemapslam_b200._capi import CslamError
    m = matcher4096
    a = _batch([bow_pair(2, 3000, 3000)])
    v2 = np.ones((1, 3000), np.uint8)
    n0, m0 = m.SearchByBoW(*a)
    k0, k12 = m.SearchByBoW_KF(a[0], a[1], a[2], a[3], a[4], a[5], v2, a[6])
    for side in (3, 6):
        b = [x.copy() for x in a]
        b[side][0, 2500] = bad
        with pytest.raises(CslamError, match=r"error -2: cslam_search_by_bow: node ids must be in \[-1, 2\^20 - 1\)"):
            m.SearchByBoW(*b)
        with pytest.raises(CslamError, match=r"error -2: cslam_search_by_bow_kf: node ids must be in \[-1, 2\^20 - 1\)"):
            m.SearchByBoW_KF(b[0], b[1], b[2], b[3], b[4], b[5], v2, b[6])
        n1, m1 = m.SearchByBoW(*a)                                        # the handle still works
        assert n1[0] == n0[0] and np.array_equal(m1, m0)
    k1, k12b = m.SearchByBoW_KF(a[0], a[1], a[2], a[3], a[4], a[5], v2, a[6])
    assert k1[0] == k0[0] and np.array_equal(k12b, k12)


# ----------------------------------------------------------------------------------------------------------------- 4. SearchForTriangulation at 4096
FACE = 650
ABSENT = (1 << 24, (1 << 24) + 1)          # the oracle's stand-ins for node -1 on KF1 / KF2: ids that never meet


def _tri_inputs(oracle, s, n1, n2, stride=STRIDE):
    """KF1 = the pair's current frame, KF2 = its observing frame, both truncated to `stride` rows; 0xAB past min(count, stride) in every
    per-feature array. Node ids 0..119 of synth.mapping_pair are mapped onto ids up to 2^20 - 2 (the mapping drop-in's sentinels included)."""
    rng = np.random.default_rng(n1 * 7 + n2)
    ids = np.concatenate([np.arange(11, 121), [*TRI_SENTINELS, *BOW_SENTINELS, 1000, 5000, 123456, 1 << 19, 777777, ID_END - 9]])
    assert len(set(ids.tolist())) == 120 and ids.max() == ID_END - 1
    idmap = rng.permutation(ids).astype(np.int32)
    kps = [s["kCur"][:stride], s["kLast"][:stride]]
    desc = [s["dCur"][:stride], s["dLast"][:stride]]
    mp = [s["hasMPCur"][:stride], s["hasMPObs"][:stride]]
    node = [idmap[s["nodeCur"][:stride]], idmap[s["nodeObs"][:stride]]]
    out = []
    for side, cnt in ((0, n1), (1, n2)):
        r = min(cnt, stride, len(kps[side]))
        assert r == min(cnt, stride)
        k = np.full(stride, 0xAB, np.uint8).repeat(kps[side].dtype.itemsize).view(kps[side].dtype)
        d = np.full((stride, 32), 0xAB, np.uint8); ry = np.full((stride, 3), 0xAB, np.uint8).repeat(4, axis=1).view(np.float32)
        h = np.full(stride, 0xAB, np.uint8); nd = np.full(stride, 0xAB, np.uint8).repeat(4).view(np.int32)
        k[:r] = kps[side][:r]; d[:r] = desc[side][:r]; ry[:r] = oracle.key_point_rays(kps[side][:r], FACE, FACE)[0]; h[:r] = mp[side][:r]; nd[:r] = node[side][:r]
        out.append([k, d, ry, h, nd, r])
    T1 = s["TcwCur"].astype(np.float64)
    Ow = (-T1[:3, :3].T @ T1[:3, 3]).astype(np.float32)
    return out[0], out[1], Ow, s["TcwLast"].reshape(16).astype(np.float32), s["E12"].reshape(9).astype(np.float32)


def _tri_oracle(oracle, s, A, B, Ow, T2, E, ori):
    r1, r2 = A[5], B[5]
    n1 = np.where(A[4][:r1] == -1, ABSENT[0], A[4][:r1]); n2 = np.where(B[4][:r2] == -1, ABSENT[1], B[4][:r2])
    return oracle.search_for_triangulation(A[0][:r1], A[1][:r1], A[2][:r1], A[3][:r1], n1, B[0][:r2], B[1][:r2], B[2][:r2], B[3][:r2], n2, Ow, T2, E,
                                           s["scale"], s["level_sigma2"], FACE, FACE, ori)


@pytest.fixture(scope="module")
def tri_pairs(oracle):
    """Six ragged pairs (n1, n2) at stride 4096, one count past the stride. In the pairs with 4096 KF2 rows: ties (a matched KF2 row copied
    to a later row of the same node) and node -1 on matched features of both sides with identical descriptors."""
    spec = [(4096, 4096), (4095, 2049), (2049, 4095), (0, 4096), (4096, 0), (5000, 4096)]
    pairs = []
    for p, (n1, n2) in enumerate(spec):
        s = synth.mapping_pair(40 + p, n=4300, faceW=FACE)
        A, B, Ow, T2, E = _tri_inputs(oracle, s, n1, n2)
        ties, absent = [], []
        if A[5] > 2048 and B[5] == STRIDE:
            rng = np.random.default_rng(500 + p)
            _, m0 = _tri_oracle(oracle, s, A, B, Ow, T2, E, False)
            i1s = np.nonzero(m0 >= 0)[0]; rng.shuffle(i1s)
            used = set(m0[m0 >= 0].tolist())
            free = [j for j in range(2100, STRIDE) if j not in used]
            rng.shuffle(free)
            for i1 in i1s[:40]:                      # tie: KF2 row i2 < 2048 copied to a later row j >= 2048 (same node, same place)
                i2 = int(m0[i1])
                if i2 >= 2048 or not free:
                    continue
                j = free.pop()
                for x in (0, 1, 2, 4):
                    B[x][j] = B[x][i2]
                B[3][j] = 0
                ties.append((int(i1), i2, j))
            for i1 in i1s[40:70]:                    # node -1 on both sides, identical descriptors: never matched
                i2 = int(m0[i1])
                A[4][i1] = -1; B[4][i2] = -1; B[1][i2] = A[1][i1]
                absent.append((int(i1), i2))
        pairs.append(dict(s=s, n=(n1, n2), A=A, B=B, Ow=Ow, T2=T2, E=E, ties=ties, absent=absent))
    return pairs


@pytest.mark.parametrize("ori", [False, True])
def test_search_for_triangulation_at_4096(oracle, tri_pairs, ori):
    from cubemapslam_b200.mapper import Mapper
    P = len(tri_pairs)
    st = lambda side, x: np.stack([t[side][x] for t in tri_pairs])
    n1 = np.array([t["n"][0] for t in tri_pairs], np.int32); n2 = np.array([t["n"][1] for t in tri_pairs], np.int32)
    s0 = tri_pairs[0]["s"]
    mapper = Mapper()
    nm, m = mapper.SearchForTriangulation(st("A", 0), st("A", 1), st("A", 2), st("A", 3), st("A", 4), n1, st("B", 0), st("B", 1), st("B", 2), st("B", 3), st("B", 4), n2,
                                          np.stack([t["Ow"] for t in tri_pairs]), np.stack([t["T2"] for t in tri_pairs]), np.stack([t["E"] for t in tri_pairs]),
                                          s0["scale"], s0["level_sigma2"], FACE, FACE, ori)
    mapper.close()
    hi1 = hi2 = 0; won = 0; nties = 0
    for p, t in enumerate(tri_pairs):
        r1 = t["A"][5]
        rn, rm = _tri_oracle(oracle, t["s"], t["A"], t["B"], t["Ow"], t["T2"], t["E"], ori)
        assert nm[p] == rn and np.array_equal(m[p, :r1], rm), "pair %d %s" % (p, t["n"])
        for i1, i2 in t["absent"]:
            assert m[p, i1] == -1
        assert not np.isin(m[p, :r1], [i2 for _, i2 in t["absent"]]).any()
        for i1, i2, j in t["ties"]:                  # the later of two equal KF2 candidates wins
            nties += 1; won += int(m[p, i1] == j)
            assert m[p, i1] != i2
        hit = rm >= 0
        if hit.any():
            hi1 = max(hi1, int(np.nonzero(hit)[0].max())); hi2 = max(hi2, int(rm[hit].max()))
        if min(r1, t["B"][5]) > 2048:
            assert rn > 100
    assert hi1 >= 2048 and hi2 >= 2048
    assert nties >= 40 and won >= 0.8 * nties * (0.5 if ori else 1)
    assert sum(len(t["absent"]) for t in tri_pairs) >= 60


# ----------------------------------------------------------------------------------------------------------------- 5. transform -> search on the device
def test_stopped_word_features_never_match_through_device_chain(oracle):
    """cslam_bow_transform_dev -> cslam_search_by_bow_dev with no host round trip, on a vocabulary with 20 % stopped words. F is the KF with a
    few bits flipped, permuted, so features on stopped words (node -1 on both sides) would match each other if node -1 were a node."""
    import torch
    from cubemapslam_b200.matcher import ORBMatcher
    from cubemapslam_b200.mapper import Mapper
    voc = balanced_tree(10, 4, seed=5, stop_frac=0.2)
    gv, _ = _voc_pair(voc, max_frames=2)
    s = synth.mapping_pair(60, n=3600, faceW=FACE)
    rng = np.random.default_rng(61)
    leaves = np.nonzero(voc["is_leaf"])[0]
    nK, nF = len(s["kLast"]), min(len(s["kCur"]), STRIDE)
    assert 3000 <= nK <= STRIDE and 3000 <= nF
    dK = voc["desc"][rng.choice(leaves, nK)] ^ _noise(rng, nK, 0.02)
    src = s["src"][:nF]
    dF = np.where((src >= 0)[:, None], dK[np.maximum(src, 0)] ^ _noise(rng, nF, 0.02), voc["desc"][rng.choice(leaves, nF)] ^ _noise(rng, nF, 0.02))
    aK = s["kLast"]["angle"].astype(np.float32); aF = s["kCur"]["angle"][:nF].astype(np.float32)
    valid = (rng.random(nK) < 0.9).astype(np.uint8)
    d = _frames_to_stride([dK, dF])
    dd = torch.from_numpy(d).cuda(); dn = torch.tensor([nK, nF], dtype=torch.int32, device="cuda")
    word, leaf, node, bw = (torch.empty((2, STRIDE), dtype=torch.int32, device="cuda") for _ in range(4))
    bv = torch.empty((2, STRIDE), dtype=torch.float64, device="cuda"); bc = torch.empty(2, dtype=torch.int32, device="cuda")
    aKd = torch.from_numpy(aK).cuda(); aFd = torch.from_numpy(aF).cuda(); vd = torch.from_numpy(valid).cuda()
    mf = torch.full((nF,), -7, dtype=torch.int32, device="cuda"); nm = torch.zeros(1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    from cubemapslam_b200._capi import check, lib, ptr
    check(lib().cslam_bow_transform_dev(gv._h, *[ptr(t.data_ptr()) for t in (dd, dn)], STRIDE, 2, 2, *[ptr(t.data_ptr()) for t in (word, leaf, node, bw, bv, bc)]))
    check(lib().cslam_vocabulary_sync(gv._h))
    m = ORBMatcher(0.7, True, max_pairs=1, max_features=STRIDE)
    row = STRIDE * 4
    m.search_by_bow_dev(dd.data_ptr(), aKd.data_ptr(), vd.data_ptr(), node.data_ptr(), nK, dd.data_ptr() + STRIDE * 32, aFd.data_ptr(), node.data_ptr() + row, nF, 1,
                        mf.data_ptr(), nm.data_ptr())
    m.sync()
    got_n, got = int(nm.cpu()[0]), mf.cpu().numpy()
    m.close(); gv.close()
    nodeK, nodeF = node[0, :nK].cpu().numpy(), node[1, :nF].cpu().numpy()
    assert 0.1 < (nodeK == -1).mean() < 0.3 and 0.1 < (nodeF == -1).mean() < 0.3
    want_n, want = oracle.search_by_bow(dK, aK, valid, np.where(nodeK == -1, BOW_SENTINELS[0], nodeK), dF, aF, np.where(nodeF == -1, BOW_SENTINELS[1], nodeF), 0.7, True)
    assert got_n == want_n and np.array_equal(got, want) and want_n > 1000
    assert np.all(got[nodeF == -1] == -1)
    # what treating -1 as one shared node would do: the test would see it
    _, shared = oracle.search_by_bow(dK, aK, valid, nodeK, dF, aF, nodeF, 0.7, True)
    assert int((shared[nodeF == -1] >= 0).sum()) > 100
    # the same node arrays through the host triangulation form (KF1 = F, KF2 = KF): accepted, and node -1 features never match
    kC, kL = s["kCur"][:nF], s["kLast"]
    rC, rL = oracle.key_point_rays(kC, FACE, FACE)[0], oracle.key_point_rays(kL, FACE, FACE)[0]
    T1 = s["TcwCur"].astype(np.float64)
    Ow = (-T1[:3, :3].T @ T1[:3, 3]).astype(np.float32); T2 = s["TcwLast"].reshape(16).astype(np.float32); E = s["E12"].reshape(9).astype(np.float32)
    hC, hL = s["hasMPCur"][:nF], s["hasMPObs"]
    for ori in (False, True):
        mapper = Mapper()
        tn, tm = mapper.SearchForTriangulation(kC[None], dF[None], rC[None], hC[None], nodeF[None], [nF], kL[None], dK[None], rL[None], hL[None], nodeK[None], [nK],
                                               Ow[None], T2[None], E[None], s["scale"], s["level_sigma2"], FACE, FACE, ori)
        mapper.close()
        rn, rm = oracle.search_for_triangulation(kC, dF, rC, hC, np.where(nodeF == -1, TRI_SENTINELS[0], nodeF), kL, dK, rL, hL,
                                                 np.where(nodeK == -1, TRI_SENTINELS[1], nodeK), Ow, T2, E, s["scale"], s["level_sigma2"], FACE, FACE, ori)
        assert tn[0] == rn and np.array_equal(tm[0], rm) and rn > 100
        assert np.all(tm[0][nodeF == -1] == -1) and np.all(nodeK[tm[0][tm[0] >= 0]] >= 0)
