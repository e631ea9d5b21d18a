"""CPU: the PoseOptimization / LocalBA oracle on the scenes of tests/pose_limits_scenes.py. The scenes must reach what they are built for
(exact thresholds, every LM stop, rejected-then-accepted trials, level changes between rounds, failed solves), and the oracle's answers are
pinned in tests/golden/refcalls_oracle_pose_limits.npz. That file records the oracle itself, to catch its drift: the BA oracle cannot be
pinned to the reference's g2o, which needs Eigen."""
import os

import numpy as np
import pytest

from tests import pose_limits_scenes as S

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "refcalls_oracle_pose_limits.npz")


def run(oracle, q, W):
    return oracle.pose_opt(q["Tcw"], q["Xw"], q["kpxy"], q["inv_sigma2"], W, W)


@pytest.mark.parametrize("W", S.WIDTHS)
def test_seams_have_no_disagreement(W):
    """face_of_pixel_f's float quotient and pos_in_face's double floor agree on every float near every seam."""
    assert len(S.seam_floats(W)) == 3 * (2 * S.SEAM_ULPS + 1)
    assert len(S.seam_disagreements(W)) == 0


@pytest.mark.parametrize("W", S.WIDTHS)
def test_stationary_frames(oracle, W):
    """Bit-unchanged identity pose, one rejected trial per round, and the pair classified by PoseOptimization's float compare."""
    for q, (wp, ev) in zip(S.stationary_frames(W), S.STATIONARY_PAIRS):
        r = run(oracle, q, W)
        assert np.array_equal(r["pose64"], [0, 0, 0, 0, 0, 0, 1])
        assert np.array_equal(r["log"][:, 2:], [[1, 0]] * 4) and np.array_equal(r["stop"], [2] * 4)
        chi = np.float64(wp) * (1 + ev * ev)
        assert (ev == 0) == (chi == np.float64(np.float32(chi)))                 # the rounding pair's chi2 is not a float
        out = np.float32(chi) > S.CHI2_TH
        assert out == (wp > S.CHI2_TH) and (chi > 5.991) == (wp >= S.CHI2_TH or ev != 0)
        assert list(r["outlier"][7:9]) == [out, out] and not r["outlier"][:7].any() and not r["outlier"][9:].any()
        assert r["inliers"] == len(q["Xw"]) - 2 * out


@pytest.mark.parametrize("W", S.WIDTHS)
def test_local_ba_classification(oracle, W):
    """LocalBA's double compare and depth test: 5.991f and one ulp above are outliers, depth 0 and -0.5 are outliers, 2^-4 is not."""
    p = S.local_ba_scene(W)
    r = oracle.local_ba(p["Tcw"], p["kf_fixed"], p["pts"], p["eMP"], p["eKF"], p["kpxy"], p["inv_sigma2"], W, W)
    assert np.array_equal(r["outlier"], p["expected"])
    assert np.array_equal(r["pts"], p["pts"]) and np.array_equal(r["log"][:, 2:], [[1, 0]] * 2)
    assert np.float64(S.CHI2_TH) > 5.991 and not np.float64(S.PAIR_WEIGHTS[2]) > 5.991


def test_off_face_rejected(oracle):
    b = S.off_face_batch(650)
    q = b[2]
    assert S.synth._pixel_to_ray(*map(float, q["kpxy"][17]), 650) is None
    with pytest.raises(ValueError, match="no cube face"):
        run(oracle, q, 650)
    few = S.frame(q["Xw"][16:18], q["kpxy"][16:18], q["inv_sigma2"][16:18])     # < 3 correspondences: returned before any edge is evaluated
    assert run(oracle, few, 650)["inliers"] == 0


def test_scenes_reach_every_case(oracle):
    """Over all widths: every way an LM round stops, a rejected trial followed by an accepted one, an edge whose level changes between rounds
    (in both directions), a frame whose first round loses every edge, and degenerate frames whose every trial is rejected."""
    stops, rej_acc, to_out, to_in, lost = set(), 0, 0, 0, 0
    for W in S.WIDTHS:
        for name, q in S.all_frames(W):
            r = run(oracle, q, W)
            stops |= set(r["stop"].tolist())
            rej_acc += int(((r["log"][:, 2] > 1) & (r["log"][:, 3] == 1)).sum())
            ro = r["round_outlier"]
            if len(q["Xw"]) >= 10:
                to_out += int((ro[1:] > ro[:-1]).sum()); to_in += int((ro[1:] < ro[:-1]).sum())
                lost += int(ro[0].all() and r["inliers"] == 0)
            if name.startswith("degenerate"):
                assert len(r["log"]) and not r["log"][:, 3].any(), (W, name)       # no solve succeeds: the kernel's x = 0 and g2o's stale x agree
        for q in S.degenerate_frames(W)[:1]:
            assert np.array_equal(run(oracle, q, W)["log"][:, 2], [10] * 4)        # H = 0, lambda = 0: ten failed solves per round
    assert stops == {0, 1, 2, 3}
    assert rej_acc > 0 and to_out > 0 and to_in > 0 and lost > 0


def answers(oracle):
    out = {}
    for W in S.WIDTHS:
        for name, q in S.all_frames(W):
            r = run(oracle, q, W)
            k = "%d_%s_" % (W, name)
            out.update({k + "inliers": np.int32(r["inliers"]), k + "outlier": r["outlier"], k + "pose64": r["pose64"], k + "log": r["log"]})
        p = S.local_ba_scene(W)
        r = oracle.local_ba(p["Tcw"], p["kf_fixed"], p["pts"], p["eMP"], p["eKF"], p["kpxy"], p["inv_sigma2"], W, W)
        out.update({"%d_localba_outlier" % W: r["outlier"], "%d_localba_log" % W: r["log"]})
    return out


def test_oracle_answers_pinned(oracle):
    got = answers(oracle)
    gold = np.load(GOLDEN)
    assert sorted(gold.files) == sorted(got)
    for k, v in got.items():
        if k.endswith("pose64") or k.endswith("log"):
            assert np.allclose(v, gold[k], rtol=1e-12, atol=0, equal_nan=True), k
        else:
            assert np.array_equal(v, gold[k]), k


if __name__ == "__main__":      # regenerate the golden file: python -m tests.test_oracle_pose_limits
    import oracle as orc
    orc.lib()
    np.savez_compressed(GOLDEN, **answers(orc))
