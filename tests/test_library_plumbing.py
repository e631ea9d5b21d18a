"""The library's shared host plumbing: no run-time tuning switches, the create-time device check of every handle, the per-kernel event
timers of the front end and the optimizer, and the micro-benchmark harness of the matcher."""
import glob
import os
import re

import numpy as np
import pytest

from cubemapslam_b200 import config, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_only_the_nccl_fallback_reads_the_environment():
    """CSLAM_BA_NCCL_ONLY forces the multi-GPU optimizer's NCCL fallback; no other environment variable changes what the library runs."""
    calls = []
    for path in glob.glob(os.path.join(ROOT, "cubemapslam_b200", "csrc", "*.cu*")):
        src = open(path).read()
        for m in re.finditer(r"\bgetenv\s*\(\s*([^)]*)\)", src):
            calls.append((os.path.basename(path), m.group(1).strip()))
    assert calls and all(arg == '"CSLAM_BA_NCCL_ONLY"' for _, arg in calls), calls


def test_device_memory_comes_from_dev_alloc_or_the_arena():
    """Persistent per-handle state is allocated by dev_alloc, everything a single call needs comes from the handle's DevArena (common.cuh).
    The one other device allocation is the multi-GPU optimizer's exchange set-up (CUDA IPC buffers and the NCCL handshake)."""
    regions = {"common.cuh": [r"static int dev_alloc\(", r"class DevArena \{"], "ba.cu": [r"static int setup_xchg\("]}
    found = {}
    for path in glob.glob(os.path.join(ROOT, "cubemapslam_b200", "csrc", "*.cu*")):
        name = os.path.basename(path)
        src = open(path).read()
        spans = []
        for start in regions.get(name, []):
            b = re.search(start, src).start()
            spans.append((start, b, re.compile(r"\n\}").search(src, b).end()))
        for m in re.finditer(r"\bcudaMalloc(?!Host)\w*\s*\(", src):
            inside = [s for s, b, e in spans if b <= m.start() < e]
            assert inside, "%s:%d allocates device memory outside dev_alloc / DevArena" % (name, src.count("\n", 0, m.start()) + 1)
            found[inside[0]] = found.get(inside[0], 0) + 1
    assert set(found) == {s for v in regions.values() for s in v}, found


def test_every_handle_needs_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("runs on the CPU-only container")
    from cubemapslam_b200 import _capi
    from cubemapslam_b200.mapper import Mapper
    from cubemapslam_b200.tracker import Tracker
    from cubemapslam_b200.vocabulary import Vocabulary
    makers = {"Tracker": Tracker, "Mapper": Mapper,
              "Vocabulary": lambda: Vocabulary(2, 1, [0, 0], [1, 1], np.zeros((2, 32), np.uint8), [1.0, 1.0])}
    for name, make in makers.items():
        with pytest.raises(_capi.CslamError) as ei:
            make()
        assert "no CUDA device" in str(ei.value), (name, str(ei.value))


@pytest.mark.gpu
def test_frontend_timing_counts_launches_and_keeps_outputs():
    """A timed batch runs on one lane; it must count every launch once and give the same bytes as the untimed two-lane batch."""
    import torch
    from cubemapslam_b200.frontend import FrontEnd
    cfg = config.front_1024()
    B = 4
    dev = torch.device("cuda", 0)
    fish = torch.from_numpy(np.stack([synth.fisheye_frame(cfg, i) for i in range(B)])).to(dev)
    fe = FrontEnd(cfg, config.load_mask("gray_cubemap_front_mask_650"), max_batch=B)
    try:
        def batch():
            kps = torch.zeros((B, fe.kp_cap, 28), dtype=torch.uint8, device=dev); desc = torch.zeros((B, fe.kp_cap, 32), dtype=torch.uint8, device=dev)
            n = torch.zeros(B, dtype=torch.int32, device=dev)
            torch.cuda.synchronize()
            fe.run_dev(fish.data_ptr(), B, kps.data_ptr(), desc.data_ptr(), n.data_ptr())
            fe.sync()
            return kps.cpu().numpy(), desc.cpu().numpy(), n.cpu().numpy()
        plain = batch()
        fe.set_timing(True)
        l0 = fe.launches
        timed = batch()
        launched = fe.launches - l0
        tm = fe.timing()
        fe.set_timing(False)
        nl = fe.nlevels
        want = {"k_warp": 1, "k_pyramid": nl - 1, "k_fast": nl, "k_distribute": 1, "k_describe": 1}
        assert {k: c for k, (_, c) in tm.items()} == want
        assert all(ms > 0 for ms, _ in tm.values()), tm
        assert launched == sum(want.values())
        assert np.array_equal(plain[2], timed[2]) and plain[2].min() > 0
        for f in range(B):
            k = plain[2][f]
            assert np.array_equal(plain[0][f, :k], timed[0][f, :k]) and np.array_equal(plain[1][f, :k], timed[1][f, :k]), "frame %d" % f
    finally:
        fe.close()


@pytest.mark.gpu
def test_optimizer_timing_runs_eagerly_with_the_graphs_results():
    """Timed LM trials run eagerly, untimed ones replay a CUDA graph: both must give the same bits."""
    from cubemapslam_b200.optimizer import Optimizer
    p = synth.ba_problem(nKF=8, nMP=300, kmin=2, kmax=6, faceW=450, seed=11, radius=1.5)
    args = (p["Tcw"], p["kf_fixed"], p["pts"], p["eMP"], p["eKF"], p["kpxy"], p["inv_sigma2"], p["faceW"], p["faceH"])
    o = Optimizer()
    try:
        graph = o.LocalBundleAdjustment(*args)
        o.set_timing(True)
        eager = o.LocalBundleAdjustment(*args)
        tm = o.timing()
        o.set_timing(False)
    finally:
        o.close()
    assert eager["trials"] > 0 and eager["trials"] == graph["trials"] and eager["iters"] == graph["iters"]
    for k in ("k_ba_solve", "k_ba_schur", "k_ba_dinv"):
        assert tm[k][1] == eager["trials"], (k, tm[k])
    for k in ("pose64", "pts64", "outlier", "log"):
        assert np.array_equal(graph[k], eager[k]), k


@pytest.mark.gpu
def test_micro_benchmarks_report_rates():
    from cubemapslam_b200.matcher import ORBMatcher
    m = ORBMatcher(max_pairs=1, max_features=256)
    try:
        for name, launches in (("ubench_popc", 2), ("ubench_minmax3", 2), ("ubench_bmma", 4)):
            l0 = m.launches
            rates = np.atleast_1d(getattr(m, name)())
            assert np.all(np.isfinite(rates)) and np.all(rates > 0), (name, rates)
            assert m.launches - l0 == launches, name
    finally:
        m.close()
