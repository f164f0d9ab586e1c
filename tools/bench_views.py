"""Throughput of tba_adjust_views (batched BundleAdjustView, one CTA per view) on cuda:0: views/s and observations/s for a
batch of 1 k and of 10 k localized views.  Each case is a seeded synthetic scene (per-camera RADTAN intrinsics with the focal
length and radial distortion free, poses disturbed, points constant); every view of the scene is in the batch.  Figures are
API-level: wall clock of the C-ABI call on the device-resident problem, including the device->host copy of the per-view results,
best of `--repeat` calls, each from the same starting parameters (tba_reset_parameters).  The first call of a case builds the
camera-major observation index and is not timed.  One JSON object on stdout."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from theiasfm_b200 import _abi, engine, synthetic  # noqa: E402


def case(n_views, obs_per_view, repeat):
    obs_per_pt = 6
    p = synthetic.make_scene(n_cam=n_views, n_pt=n_views * obs_per_view // obs_per_pt, obs_per_pt=obs_per_pt, seed=n_views,
                             model=_abi.MODEL_PINHOLE_RADIAL_TANGENTIAL, shared_intrinsics=False)
    p.pt_const[:] = 1
    kw = dict(use_inner_iterations=0, linear_solver_type=_abi.DENSE_QR, max_num_iterations=50)
    views = np.arange(p.n_cam, dtype=np.int32)
    eng = engine.Engine()
    eng.upload(p, engine.default_options(**kw))
    eng.adjust_views(engine.default_options(**kw), views)     # warm-up: modules, camera-major index
    best, it = float("inf"), None
    for _ in range(repeat):
        eng.reset_parameters(p)
        t = time.perf_counter()
        st, ic, fc, it = eng.adjust_views(engine.default_options(**kw), views)
        best = min(best, time.perf_counter() - t)
    eng.close()
    return dict(views=int(p.n_cam), observations=int(p.n_obs), seconds=best, views_per_s=p.n_cam / best, obs_per_s=p.n_obs / best,
                mean_lm_iterations=float(np.mean(it)), converged=int((st == _abi.CONVERGENCE).sum()), failed=int((st == _abi.FAILURE).sum()))


def main():
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument("--obs-per-view", type=int, default=600)
    ap.add_argument("--repeat", type=int, default=5)
    a = ap.parse_args()
    if engine.device_count() < 1:
        sys.exit("bench_views: no CUDA device (this tool measures the GPU only)")
    import subprocess
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    out = dict(gpu=gpu, cases=[case(n, a.obs_per_view, a.repeat) for n in (1000, 10000)])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
