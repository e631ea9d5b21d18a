"""GPU: LocalBundleAdjustment against the oracle on the scenes of tests/local_ba_limits_scenes.py, at every face width, on one reused
Optimizer handle. Exact: iterations, trials, the LM log's trials / accepted columns, outlier flags; chi2 and lambda to 1e-8 relative (NaN where
the oracle has NaN); pose64 and pts64 to 1e-5 relative, bit-identical on the stationary scene. The NaN-lambda scenes also run through the
landmark-sharded path where the box has two GPUs."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import local_ba_limits_scenes as S

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def opt():
    from cubemapslam_b200.optimizer import Optimizer
    o = Optimizer()
    yield o
    o.close()


def rel(a, b):
    return np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


@pytest.mark.parametrize("W", S.WIDTHS)
def test_local_ba_limits(oracle, opt, W):
    for name, p in S.all_scenes(W):
        r = oracle.local_ba(*S.args(p), **S.kwargs(p))
        g = opt.LocalBundleAdjustment(*S.args(p), **S.kwargs(p))
        assert g["iters"] == r["iters"] and g["trials"] == int(r["log"][:, 2].sum()), (name, g["iters"], r["iters"], g["trials"])
        assert np.array_equal(g["log"][:, 2:], r["log"][:, 2:]), name
        assert np.allclose(g["log"][:, :2], r["log"][:, :2], rtol=1e-8, atol=0, equal_nan=True), name
        assert np.array_equal(g["outlier"], r["outlier"]), (name, np.flatnonzero(g["outlier"] != r["outlier"]))
        assert rel(g["pose64"], r["pose64"]) < 1e-5 and rel(g["pts64"], r["pts64"]) < 1e-5, name
        if name == "stationary":
            assert np.array_equal(bits(g["pose64"]), bits(r["pose64"])) and np.array_equal(bits(g["pts64"]), bits(r["pts64"]))
            assert np.array_equal(g["pts"], p["pts"]) and np.array_equal(g["Tcw"], p["Tcw"])


def test_nan_lambda_sharded():
    """The NaN-lambda scenes through the landmark-sharded path (two ranks) match the single-GPU run: LM decisions and outliers exactly, chi2
    and lambda to 1e-8, state to 1e-5 (the ranks add their partial sums in another order than one GPU)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1", "--master-port", "29613",
           os.path.join(ROOT, "tools", "ba_multi_gpu.py"), "nan_lambda"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
    d = json.loads([line for line in out.stdout.splitlines() if line.startswith("{")][-1])
    assert d["scenes"] == 9 and d["all_match"], d
