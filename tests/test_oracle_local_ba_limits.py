"""CPU: the LocalBA oracle on the scenes of tests/local_ba_limits_scenes.py. The scenes must reach what they are built for (every way a round
ends, in both rounds; NaN lambda; failed solves; second rounds whose active set shrinks; stale and fresh chi2 on both sides of 5.991; the stop
flag after accepted and rejected trials), and the oracle's answers are pinned in tests/golden/refcalls_oracle_local_ba_limits.npz. That file
records the oracle itself, to catch its drift: the BA oracle cannot be pinned to the reference's g2o, which needs Eigen."""
import os

import numpy as np
import pytest

from tests import local_ba_limits_scenes as S

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "refcalls_oracle_local_ba_limits.npz")
KEYS = ("outlier", "pose64", "pts64", "log", "round", "stop", "level", "chi2")


def run(oracle, p, **kw):
    return oracle.local_ba(*S.args(p), **{**S.kwargs(p), **kw})


def fresh_chi2(oracle, p, r):
    return oracle.ba_edge_chi2(r["pose64"], r["pts64"], p["eMP"], p["eKF"], p["kpxy"], p["inv_sigma2"], p["faceW"], p["faceH"])


def depth(r, p):
    """Camera-frame depth of every edge's MapPoint at the final fp64 state (pose64: t, qx qy qz qw)."""
    t, q, X = r["pose64"][p["eKF"], :3], r["pose64"][p["eKF"], 3:], r["pts64"][p["eMP"]]
    uv = 2 * np.cross(q[:, :3], X)
    return (X + q[:, 3:] * uv + np.cross(q[:, :3], uv) + t)[:, 2]


def diagonals(oracle, p, pts=None):
    """g2o's index-mapping order of LocalBA's first linearisation at the input state (robust kernel on): the six diagonals of every free
    pose, then the three of every MapPoint, as |H_jj| per vertex (pose rows first). Every vertex must have an edge."""
    W = p["faceW"]; pts = p["pts"] if pts is None else pts
    d = float(np.float32(np.sqrt(5.991))); d2 = d * d
    Hp = {k: np.zeros(6) for k in np.flatnonzero(p["kf_fixed"] == 0)}
    Hl = np.zeros((len(pts), 3))
    for e in range(len(p["eMP"])):
        k, l = p["eKF"][e], p["eMP"][e]
        err, Jp, Jx, _ = oracle.edge_eval(p["Tcw"][k], pts[l].astype(np.float64), p["kpxy"][e, 0], p["kpxy"][e, 1], W, W)
        w = float(p["inv_sigma2"][e]); c = w * (err @ err)
        w *= 1.0 if c <= d2 else d / np.sqrt(c)
        Hl[l] += w * (Jx ** 2).sum(0)
        if k in Hp:
            Hp[k] += w * (Jp ** 2).sum(0)
    return [Hp[k] for k in sorted(Hp)], Hl


@pytest.mark.parametrize("W", S.WIDTHS)
def test_stationary(oracle, W):
    """b = 0 exactly: one trial per round, rho == 0, poses and points bit-identical to the input; the 5.991f pairs leave round 2."""
    p = S.stationary(W)
    r = run(oracle, p)
    assert np.array_equal(r["log"][:, 2:], [[1, 0]] * 2) and np.array_equal(r["stop"], [2, 2]) and np.array_equal(r["round"], [0, 1])
    assert np.array_equal(r["pts64"], p["pts"].astype(np.float64)) and np.array_equal(r["pose64"], np.tile([0, 0, 0, 0, 0, 0, 1.0], (3, 1)))
    assert r["level"].any() and r["log"][1, 0] < r["log"][0, 0]


@pytest.mark.parametrize("W", S.WIDTHS)
def test_nan_lambda(oracle, W):
    """The face-plane MapPoint seen by a fixed key frame: lambda NaN through round 1 when it is the last vertex, finite when it is first or
    in the middle (the maximum over the vertices after it); seen by the free key frame, every trial of round 1 is one failed solve."""
    for where in ("first", "middle", "last"):
        p = S.plane_fixed(W, where)
        r = run(oracle, p)
        lam = r["log"][r["round"] == 0, 1]
        assert np.isinf(r["log"][0, 0])
        assert np.isnan(lam).all() if where == "last" else np.isfinite(lam).all(), where
        if where != "last":
            # lambda_0 = 1e-5 x the largest diagonal AFTER the NaN one: the free pose's larger diagonal drops out (a NaN-skipping max keeps it)
            plane = int(np.flatnonzero((p["pts"] == np.float32(S.PLANE[0])).all(1))[0])
            Hp, Hl = diagonals(oracle, p)
            after = np.abs(Hl[plane + 1:]).max()
            assert np.array_equal(r["log"][0, 2:], [1, 0])                   # row 0 is one rejected trial: lambda_0 doubled once
            assert np.isclose(r["log"][0, 1] / 2, 1e-5 * after, rtol=1e-9, atol=0), where
            assert np.abs(Hp[0]).max() > after
    r = run(oracle, S.plane_free(W))
    one = r["round"] == 0
    assert np.array_equal(r["log"][one, 2:], [[1, 0]] * 5) and np.isinf(r["log"][one, 0]).all()


@pytest.mark.parametrize("W", S.WIDTHS)
def test_failed_solves(oracle, W):
    """Every weight 0: ten failed solves per round, lambda 0. Zero-weight round 2: the landmarks moved in round 1, round 2 is ten failed
    solves and leaves the state of round 1; every edge an outlier: round 2 runs no iteration."""
    r = run(oracle, S.zero_weight(W))
    assert np.array_equal(r["log"][:, 1:], [[0, 10, 0]] * 2) and np.array_equal(r["stop"], [1, 1])
    p = S.conflicting(W)
    r, r1 = run(oracle, p), run(oracle, p, its2=0)
    two = r["round"] == 1
    assert np.array_equal(r["log"][two, 1:], [[0, 10, 0]]) and r["stop"][-1] == 1
    moved = p["inv_sigma2"] > 0
    assert (r["level"] == moved).all() or (r["level"][moved]).all()
    assert not np.array_equal(r1["pts64"], p["pts"].astype(np.float64))
    assert np.array_equal(r["pts64"], r1["pts64"]) and np.array_equal(r["pose64"], r1["pose64"])
    q = S.conflicting(W, False)
    r = run(oracle, q)
    assert r["level"].all() and (r["round"] == 0).all() and r["outlier"].all()


@pytest.mark.parametrize("W", S.WIDTHS)
def test_second_round_active_set(oracle, W):
    """A landmark whose every edge is an outlier keeps its round-1 position and is flagged from its round-1 error; a free key frame that
    loses every edge keeps its round-1 pose."""
    for name, p in [("lost_keyframe", S.lost_keyframe(W))] + [s for s in S.schedule(W) if s[0].endswith("_5_10")]:
        r, r1 = run(oracle, p), run(oracle, p, its2=0)
        assert r1["iters"] == p.get("its1", 5) or r1["stop"][-1] != 0
        gone = [l for l in range(len(p["pts"])) if (r["level"][p["eMP"] == l] == 1).all() and (p["eMP"] == l).any()]
        for l in gone:
            assert np.array_equal(r["pts64"][l], r1["pts64"][l]), (name, l)
        e = np.isin(p["eMP"], gone)
        assert np.array_equal(r["chi2"][e], r1["chi2"][e]), name
        if name == "lost_keyframe":
            assert (r["level"][p["eKF"] == 2] == 1).all() and (r["level"][p["eKF"] == 3] == 0).any()
            assert np.array_equal(r["pose64"][2], r1["pose64"][2]) and len(gone) > 0


@pytest.mark.parametrize("W", S.WIDTHS)
def test_stop_flag(oracle, W):
    stops = dict(S.stop_scenes(W))
    base, r = run(oracle, stops["stop_past_end"], stop_after_trials=0), run(oracle, stops["stop_past_end"])
    for key in KEYS:
        assert np.array_equal(r[key], base[key], equal_nan=True), key
    r = run(oracle, stops["stop_accepted"])
    assert r["stop"][-1] == 4 and r["log"][-1, 3] == 1 and (r["round"] == 0).all() and not r["level"].any()
    r = run(oracle, stops["stop_round2"])
    assert r["stop"][-1] == 4 and r["round"][-1] == 1
    p = stops["stop_rejected"]
    r = run(oracle, p)
    assert r["stop"][-1] == 4 and r["log"][-1, 3] == 0 and (r["round"] == 0).all() and not r["level"].any()
    assert np.array_equal(r["log"][:, 2:], [[1, 1], [1, 1], [1, 0]]) and S.STRADDLE_K == 3
    fresh = fresh_chi2(oracle, p, r)
    straddle = (r["chi2"] > 5.991) != (fresh > 5.991)
    assert np.flatnonzero(straddle).tolist() == [S.STRADDLE_EDGE]
    e = S.STRADDLE_EDGE
    assert r["chi2"][e] > 1.2 * 5.991 and fresh[e] < 5.991 / 1.2 and r["outlier"][e] == 1     # flagged from the rejected trial's error
    behind = ~(depth(r, p) > 0)
    assert np.array_equal(r["outlier"], (r["chi2"] > 5.991) | behind)


def test_scenes_reach_every_case(oracle):
    """Over all widths: every stop code in each round, a trial loop that ends on a rejected trial after an accepted one, an outlier whose
    round-1 chi2 is above 5.991 and whose chi2 at the final state is below (the reference still flags it)."""
    stops = {0: set(), 1: set()}
    rej_acc, stale = 0, 0
    for W in S.WIDTHS:
        for name, p in S.all_scenes(W):
            r = run(oracle, p)
            for rd, st in zip(r["round"], r["stop"]):
                stops[int(rd)].add(int(st))
            rej_acc += int(((r["log"][:, 2] > 1) & (r["log"][:, 3] == 1)).sum())
            if "stop" not in name:
                fresh = fresh_chi2(oracle, p, r)
                s = (r["level"] == 1) & (r["chi2"] > 5.991) & (fresh < 5.991)
                assert (r["outlier"][s] == 1).all()
                stale += int(s.sum())
    assert stops[0] == {0, 1, 2, 3, 4} and stops[1] == {0, 1, 2, 3, 4}, stops
    assert rej_acc > 0 and stale > 0


def answers(oracle):
    out = {}
    for W in S.WIDTHS:
        for name, p in S.all_scenes(W):
            r = run(oracle, p)
            out.update({"%d_%s_%s" % (W, name, k): r[k] for k in KEYS})
            out["%d_%s_iters" % (W, name)] = np.int32(r["iters"])
    return out


def test_oracle_answers_pinned(oracle):
    got = answers(oracle)
    gold = np.load(GOLDEN)
    assert sorted(gold.files) == sorted(got)
    for k, v in got.items():
        if k.endswith(("pose64", "pts64", "log", "chi2")):
            assert np.allclose(v, gold[k], rtol=1e-12, atol=0, equal_nan=True), k
        else:
            assert np.array_equal(v, gold[k]), k


if __name__ == "__main__":      # regenerate the golden file: python -m tests.test_oracle_local_ba_limits
    import oracle as orc
    orc.lib()
    np.savez_compressed(GOLDEN, **answers(orc))
