#!/usr/bin/env python
"""The reference's pipeline driver `scripts/run_phys_mocap.py` (kinematic initialisation -> phys-optim inputs -> physics-based
optimisation -> results back on the skeleton), in one process and with ONE batched physics solve over all videos instead
of a `./phys_optim` process per clip.

    python scripts/run_phys_mocap.py --data <dir of video dirs> --character combined --skel_path <combined skeleton .bvh>

Every `<data>/<video>/` holds `openpose_result/*.json`, `tracked_results.json` (Monocular Total Capture) and
`foot_contacts.npy` (scripts/detect_contacts.py).  Written per video, as the reference does: `kinematic_results/{foot_contacts.npy,
floor_out.txt, final_test.bvh, <character>_out.bvh}`, `phys_optim_in_<character>/*.txt`, `phys_optim_out_<character>/{sol_out_*.txt,
success_log.txt, <video>_<character>_{no_dynamics,dynamics,durations}.bvh}`.
The frame rate comes from --fps (the reference reads it from the mp4 with OpenCV, which this image does not have).
Characters: `combined` (the video's own skeleton) and `ybot` (re-targeted with `chd.results.retarget`; needs --character_skel,
the character's skeleton .bvh -- the reference ships skeleton_fitting/ybot.bvh); `ty` / `skeletonzombie` have no table here."""
import argparse
import glob
import os
import shutil
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--data", required=True)
    ap.add_argument("--character", default="combined", choices=["combined", "ybot", "ty", "skeletonzombie"])
    ap.add_argument("--kinematic_gt_floor", action="store_true")
    ap.add_argument("--kinematic_viz", action="store_true")
    ap.add_argument("--towr_phys_optim_path", default=None, help="ignored: the solver is libchd")
    ap.add_argument("--skel_path", required=True, help="the 28-joint combined skeleton (the reference ships skeleton_fitting/combined_body_25.bvh)")
    ap.add_argument("--character_skel", default=None, help="skeleton .bvh of the character (re-targeting), e.g. skeleton_fitting/ybot.bvh")
    ap.add_argument("--fps", type=float, default=30.0)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args(argv)
    import chd
    if a.character not in chd.prepare.CHARACTERS:
        sys.exit("no character table for '%s' in this build (combined, ybot)" % a.character)
    if a.character != "combined" and not a.character_skel:
        sys.exit("--character_skel <skeleton .bvh of %s> is needed for re-targeting" % a.character)
    from chd import io_formats
    info = chd.prepare.CHARACTERS[a.character]()
    vids = sorted(d for d in os.listdir(a.data) if os.path.isdir(os.path.join(a.data, d)) and d[0] != ".")
    if not vids:
        sys.exit("No video directories in the data path!")
    dev = "cuda:%d" % a.device
    problems, meta = [], []
    secs = {"kinematic": 0.0, "physics": 0.0, "apply": 0.0}   # wall time per stage of the pipeline, all videos
    for v in vids:
        vd = os.path.join(a.data, v)
        n = len(glob.glob(os.path.join(vd, "openpose_result", "*.json")))
        kin = os.path.join(vd, "kinematic_results")
        print("Running kinematic optimization for %s (%d frames)..." % (v, n))
        t0 = time.time()
        chd.kinopt.optimize_2d_3d(os.path.join(vd, v + ".mp4"), a.skel_path, kin, 0, n, a.kinematic_gt_floor, device=dev)
        char_bvh = os.path.join(kin, a.character + "_out.bvh")
        if a.character == "combined":
            shutil.copyfile(os.path.join(kin, "final_test.bvh"), char_bvh)
        else:
            print("Running retargeting...")
            chd.results.retarget(os.path.join(kin, "final_test.bvh"), a.character_skel, info, char_bvh, device=dev)
        pin = os.path.join(vd, "phys_optim_in_" + a.character)
        os.makedirs(pin, exist_ok=True)
        print("Generating input for physics-based optimization...")
        p = chd.prepare.prepare_input(char_bvh, os.path.join(kin, "floor_out.txt"), os.path.join(kin, "foot_contacts.npy"), pin, info, 0, n,
                                      1.0 / a.fps, False, device=dev)
        problems.append(io_formats.read_phys_inputs(pin, n))      # through the files, like the reference's binary
        meta.append((v, vd, n, char_bvh))
        secs["kinematic"] += time.time() - t0
    print("Running physics-based optimization (%d sequences, one batch)..." % len(problems))
    t0 = time.time()
    with chd.phys.PhysBatch(problems, device=a.device) as batch:
        out = batch.solve()
    secs["physics"] = time.time() - t0
    t0 = time.time()
    for i, (v, vd, n, char_bvh) in enumerate(meta):
        pout = os.path.join(vd, "phys_optim_out_" + a.character)
        os.makedirs(pout, exist_ok=True)
        chd.phys.write_outputs(out, i, problems[i], pout)
        for tag in ("no_dynamics", "dynamics", "durations"):
            res = chd.results.load_towr_results(os.path.join(pout, "sol_out_%s.txt" % tag))
            anim, names, _, _ = chd.results.apply_results(res, char_bvh, 0, n, info, run_ik=True, device=dev)
            if info.heel_inds is None and res.feet_pos.shape[1] == 4:
                anim = chd.results.remove_heel_from_anim(anim)                      # towr_utils.py:972-974
            chd.results.save_bvh(os.path.join(pout, "%s_%s_%s.bvh" % (v, a.character, tag)), anim, anim.names)
        print("%s: dynamics %d durations %d" % (v, out["success"][i, 0], out["success"][i, 1]))
    secs["apply"] = time.time() - t0
    print("wall time: kinematic %.1f s (with the phys-optim inputs), physics %.1f s, apply %.1f s (with the .bvh files)" % (
        secs["kinematic"], secs["physics"], secs["apply"]))


if __name__ == "__main__":
    main()
