"""Generates tests/golden/fountain11_ir.npz from the reference's own fixtures in a TheiaSfM checkout
  <theia>/data/sfm/fountain11.bin      (a reconstruction saved by Theia after ITS OWN bundle adjustment)
  <theia>/data/sfm/gt_fountain11.bin   (ground-truth cameras of Strecha fountain-P11)
used by incremental_reconstruction_estimator_test.cc:52-160.  The reference cannot run here (C++ needing Ceres), but its
saved OUTPUT travels: the flattened IR of that reconstruction pins our cost function against a state the reference's
BA produced (tests/test_fountain_fixture.py).    Run:  python tests/golden/make_fountain_fixture.py <theia checkout>
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import theia_cereal  # noqa: E402

def main():
    DATA = os.path.join(sys.argv[1], "data", "sfm")
    rec = theia_cereal.reconstruction(open(os.path.join(DATA, "fountain11.bin"), "rb").read())
    gt = theia_cereal.reconstruction(open(os.path.join(DATA, "gt_fountain11.bin"), "rb").read())
    assert rec["consumed"] == rec["total"] and gt["consumed"] == gt["total"]
    vids = sorted(rec["views"])
    tids = sorted(t for t in rec["tracks"] if rec["tracks"][t]["est"])
    assert all(rec["views"][v]["est"] for v in vids)
    cam_of = {v: i for i, v in enumerate(vids)}
    pt_of = {t: i for i, t in enumerate(tids)}
    names = [rec["views"][v]["name"] for v in vids]
    ext = np.array([rec["views"][v]["camera"]["ext"] for v in vids])
    assert len({rec["views"][v]["camera"]["intr_id"] for v in vids}) == 1  # one shared PinholeCameraModel
    intr = np.zeros((1, 10))
    intr[0, :7] = rec["views"][vids[0]]["camera"]["intr"]
    pt = np.array([rec["tracks"][t]["pt"] for t in tids])
    oc, op, oxy = [], [], []
    for v in vids:
        for t, f in sorted(rec["views"][v]["features"].items()):
            if t in pt_of:
                oc.append(cam_of[v]); op.append(pt_of[t]); oxy.append(f)
    gt_by_name = {gt["views"][v]["name"]: gt["views"][v]["camera"] for v in gt["views"]}
    gt_ext = np.array([gt_by_name[n]["ext"] for n in names])
    gt_intr = np.array([gt_by_name[n]["intr"] for n in names])
    out = os.path.join(HERE, "fountain11_ir.npz")
    np.savez_compressed(out, names=np.array(names), ext=ext, intr=intr, pt=pt, obs_cam=np.array(oc, np.int32),
                        obs_pt=np.array(op, np.int32), obs_xy=np.array(oxy), gt_ext=gt_ext, gt_intr=gt_intr)
    print("wrote", out, "cams", len(vids), "points", len(tids), "obs", len(oc), "bytes", os.path.getsize(out))


if __name__ == "__main__":
    main()
