"""Landmark-sharded LocalBA over NCCL: run under torchrun (one rank per GPU); every rank solves the same window, rank r owns
landmarks l % N == r, the reduced camera system is all-reduced inside libcubemap_b200.so. Rank 0 checks the result against a
single-GPU run of the same problem and prints one JSON line."""
import json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist
from cubemapslam_b200 import synth
from cubemapslam_b200.optimizer import Optimizer

rank = int(os.environ.get("RANK", "0")); world = int(os.environ.get("WORLD_SIZE", "1")); local = int(os.environ.get("LOCAL_RANK", "0"))
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
small = len(sys.argv) > 1 and sys.argv[1] == "small"
if len(sys.argv) > 1 and sys.argv[1] == "nan_lambda":
    # the face-plane scenes of tests/local_ba_limits_scenes.py (NaN lambda, and the maxima after a NaN diagonal) on every rank; rank 0 compares
    # the sharded result with a single-GPU run. The ranks sum chi2 and the pose blocks in another order than one GPU does, so only the LM
    # decisions and the outliers are exact; chi2 and lambda agree to 1e-8 (NaN where NaN), poses and points to 1e-5 overall
    from tests import local_ba_limits_scenes as S
    o = Optimizer(device=local)
    idt = torch.zeros(128, dtype=torch.uint8, device="cuda")
    if rank == 0:
        idt.copy_(torch.from_numpy(Optimizer.nccl_unique_id()))
    dist.broadcast(idt, 0)
    o.init_nccl(idt.cpu().numpy(), rank, world)
    ref = Optimizer(device=local) if rank == 0 else None
    n, same = 0, True
    for W in S.WIDTHS:
        for where in ("first", "middle", "last"):
            a = S.args(S.plane_fixed(W, where))
            g = o.LocalBundleAdjustment(*a)
            if rank == 0:
                r = ref.LocalBundleAdjustment(*a)
                rl = lambda a, b: float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))
                same &= bool(g["iters"] == r["iters"] and np.array_equal(g["log"][:, 2:], r["log"][:, 2:]) and np.array_equal(g["outlier"], r["outlier"])
                             and np.allclose(g["log"][:, :2], r["log"][:, :2], rtol=1e-8, atol=0, equal_nan=True)
                             and rl(g["pose64"], r["pose64"]) < 1e-5 and rl(g["pts64"], r["pts64"]) < 1e-5)
            n += 1
    if rank == 0:
        print(json.dumps({"n_gpus": world, "scenes": n, "all_match": same}))
    dist.destroy_process_group()
    sys.exit(0)
dense = len(sys.argv) > 1 and sys.argv[1] == "dense"
prof = "prof" in sys.argv[1:]
p = (synth.ba_problem(nKF=12, nMP=1500, kmin=2, kmax=8, faceW=450, seed=3, radius=1.5) if small else
     synth.ba_problem(nKF=50, nMP=4000, kmin=50, kmax=50, radius=9.0) if dense else synth.ba_problem())
W = p["faceW"]
args = (p["Tcw"], p["kf_fixed"], p["pts"], p["eMP"], p["eKF"], p["kpxy"], p["inv_sigma2"], W, W)
o = Optimizer(device=local)
idt = torch.zeros(128, dtype=torch.uint8, device="cuda")
if rank == 0:
    idt.copy_(torch.from_numpy(Optimizer.nccl_unique_id()))
dist.broadcast(idt, 0)
o.init_nccl(idt.cpu().numpy(), rank, world)
o.LocalBundleAdjustment(*args, its1=1, its2=0)      # warm-up (NCCL channels, allocations)
dist.barrier(); torch.cuda.synchronize()
t0 = time.perf_counter()
g = o.LocalBundleAdjustment(*args)
torch.cuda.synchronize(); dist.barrier()
dt = time.perf_counter() - t0
tt = torch.tensor([dt], dtype=torch.float64, device="cuda"); dist.all_reduce(tt, op=dist.ReduceOp.MAX)
if prof:   # per-kernel CUDA-event timing of one more call (every rank takes part; rank 0 prints)
    o.set_timing(True)
    o.LocalBundleAdjustment(*args)
    tm = o.timing(); o.set_timing(False)
    if rank == 0:
        tot = sum(v[0] for v in tm.values())
        for k, (ms, cnt) in sorted(tm.items(), key=lambda kv: -kv[1][0]):
            print(f"  {k:16s} {1e3 * ms / max(cnt, 1):8.1f} us avg over {cnt:3d}  ({100 * ms / tot:4.1f}%)", file=sys.stderr)
        print(f"  GPU time per LM trial (events), rank 0 of {world}: {1e3 * tot / max(g['trials'] if 'trials' in g else g['iters'], 1):.1f} us", file=sys.stderr)
if rank == 0:
    ref = Optimizer(device=local)
    r = ref.LocalBundleAdjustment(*args)
    rel = lambda a, b: float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))
    out = {"n_gpus": world, "edges": int(len(p["eMP"])), "lm_iters": int(g["iters"]), "lm_iters_single": int(r["iters"]), "seconds": round(float(tt.item()), 4),
           "lm_iters_per_s": round(g["iters"] / float(tt.item()), 2), "rel_pose_vs_single_gpu": rel(g["pose64"], r["pose64"]),
           "rel_points_vs_single_gpu": rel(g["pts64"], r["pts64"]), "outliers_equal": bool(np.array_equal(g["outlier"], r["outlier"])),
           "log_equal": bool(np.array_equal(g["log"][:, 2:], r["log"][:, 2:]))}
    print(json.dumps(out))
    assert out["rel_pose_vs_single_gpu"] < 1e-5 and out["rel_points_vs_single_gpu"] < 1e-5 and out["outliers_equal"], out
dist.destroy_process_group()
