"""Generates the contact-classifier golden vectors by running the REFERENCE's own code
(src/contact_learning of a checkout of the reference at $CHD_REFERENCE_DIR, default ../contact-human-dynamics next to
this repository: RealVideoDataset, OpenPoseModel, test.val_full_video) on small synthetic OpenPose directories with
seeded weights.  Run once; the outputs under tests/golden/contact/ are committed, so the tests need no reference.

    python tests/golden/make_contact_golden.py

Viz-only imports the reference pulls in (skimage, matplotlib) are stubbed; np.int is aliased (test.py:107,151 use the
removed alias).  Nothing from the reference is copied into the repo: only its inputs/outputs are stored.
"""
import json
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = os.path.join(os.environ.get("CHD_REFERENCE_DIR", os.path.join(ROOT, "..", "contact-human-dynamics")), "src")


def contact_weights(seed=0):
    """Deterministic (numpy) stand-in for the unavailable pretrained weights: xavier-like Linear weights, non-trivial
    BatchNorm running statistics.  Key names follow the reference state_dict (model.{0,1,3,4,6,7,10,11,13}.*)."""
    rng = np.random.default_rng(seed)
    dims = [351, 1024, 512, 128, 32, 20]
    lin_ids, bn_ids = [0, 3, 6, 10, 13], [1, 4, 7, 11]
    sd = {}
    for li, (i, o) in zip(lin_ids, zip(dims[:-1], dims[1:])):
        a = np.sqrt(6.0 / (i + o))
        sd["model.%d.weight" % li] = rng.uniform(-a, a, (o, i)).astype(np.float32)
        sd["model.%d.bias" % li] = rng.normal(0, 0.05, o).astype(np.float32)
    for bi, o in zip(bn_ids, dims[1:-1]):
        sd["model.%d.weight" % bi] = rng.uniform(0.5, 1.5, o).astype(np.float32)
        sd["model.%d.bias" % bi] = rng.normal(0, 0.1, o).astype(np.float32)
        sd["model.%d.running_mean" % bi] = rng.normal(0, 0.1, o).astype(np.float32)
        sd["model.%d.running_var" % bi] = rng.uniform(0.5, 1.5, o).astype(np.float32)
        sd["model.%d.num_batches_tracked" % bi] = np.array(100, dtype=np.int64)
    return sd


def synth_keypoints(seed, n_frames):
    """BODY_25 keypoints of a walking stick figure at 1920x1080 with confidence drop-outs (SURVEY 8(d))."""
    rng = np.random.default_rng(seed)
    t = np.arange(n_frames) / 30.0
    kp = np.zeros((n_frames, 25, 3))
    cx = 400 + 300 * t + rng.normal(0, 1.0, n_frames)
    cy = 520 + 8 * np.sin(2 * np.pi * 2 * t)
    base = rng.normal(0, 60, (25, 2))
    base[8] = 0
    for j in range(25):
        ph = rng.uniform(0, 2 * np.pi)
        kp[:, j, 0] = cx + base[j, 0] + 25 * np.sin(2 * np.pi * 1.0 * t + ph)
        kp[:, j, 1] = cy + base[j, 1] + 120 * (j in (10, 11, 13, 14, 19, 20, 21, 22, 23, 24)) + 15 * np.cos(2 * np.pi * 1.0 * t + ph)
    kp[:, :, :2] += rng.normal(0, 1.5, (n_frames, 25, 2))
    kp[:, :, 2] = rng.uniform(0.3, 1.0, (n_frames, 25))
    # low-confidence runs of 1..5 frames, including leading / trailing runs
    for j in range(25):
        f = 0
        while f < n_frames:
            if rng.uniform() < 0.05:
                L = int(rng.integers(1, 6))
                kp[f:f + L, j, 2] = rng.uniform(0.0, 0.19, min(L, n_frames - f))
                f += L
            f += 1
    kp[:3, 11, 2] = 0.05      # leading run
    kp[-2:, 22, 2] = 0.1      # trailing run
    kp[:, 3, 2] = 0.01        # a joint that is never confident
    return kp


def write_openpose_dir(path, kp):
    os.makedirs(path, exist_ok=True)
    for f in range(kp.shape[0]):
        d = {"version": 1.3, "people": [{"pose_keypoints_2d": [float(x) for x in kp[f].reshape(-1)]}]}
        if f == 5 and kp.shape[0] > 45:   # a frame without detections -> zeros (openpose_utils.py:60-62)
            d = {"version": 1.3, "people": []}
        with open(os.path.join(path, "frame_%012d_keypoints.json" % f), "w") as fh:
            json.dump(d, fh)


def main():
    for name in ["skimage", "skimage.io", "skimage.transform", "matplotlib", "matplotlib.pyplot", "matplotlib.animation",
                 "matplotlib.patheffects", "mpl_toolkits", "mpl_toolkits.mplot3d", "torchvision", "torchvision.transforms",
                 "torchvision.utils", "cv2"]:
        if name not in sys.modules:
            try:
                __import__(name)
            except Exception:
                sys.modules[name] = types.ModuleType(name)
    np.int = int
    import torch
    os.chdir(REF)
    for p in ["contact_learning", ".", "utils", "optimize"]:
        sys.path.insert(0, os.path.join(REF, p))
    from models.openpose_only import OpenPoseModel
    from data.real_video_dataset import RealVideoDataset
    import test as ref_test
    from torch.utils.data import DataLoader

    out_dir = os.path.join(HERE, "contact")
    os.makedirs(out_dir, exist_ok=True)
    lens = {"vid_a": 57, "vid_b": 41, "vid_c": 64}
    with tempfile.TemporaryDirectory() as tmp:
        raw = {}
        for i, (name, F) in enumerate(lens.items()):
            kp = synth_keypoints(100 + i, F)
            raw[name] = kp
            write_openpose_dir(os.path.join(tmp, "data", name, "openpose_result"), kp)
        ds = RealVideoDataset(os.path.join(tmp, "data"), split="test", window_size=9, contact_size=5, load_img=False,
                              use_confidence=True, joint_set="lower")
        model = OpenPoseModel(9, 13, 5, 3)
        sd = contact_weights(0)
        model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
        model.eval()
        bs = ds.get_num_test_windows_per_seq()
        loader = DataLoader(ds, batch_size=bs, shuffle=False, num_workers=0)
        # logits of every window (reference forward, torch CPU fp32)
        logits = []
        windows = []
        with torch.no_grad():
            for batch in loader:
                windows.append(batch["joint2d"].numpy())
                logits.append(model(batch["joint2d"]).numpy())
        res = os.path.join(tmp, "out")
        with torch.no_grad():
            ref_test.val_full_video(loader, ds, model, torch.device("cpu"), 0.5, 5, contacts_out_path=res)
        contacts = {n: np.load(os.path.join(res, n, "foot_contacts.npy")) for n in lens}
        np.savez_compressed(os.path.join(out_dir, "contact_golden.npz"),
                            names=np.array(sorted(lens)), seq_lens=np.array([lens[n] for n in sorted(lens)]),
                            **{"raw_" + n: raw[n] for n in lens},
                            **{"proc_" + n: ds.op_data[i] for i, n in enumerate(sorted(lens))},
                            windows=np.stack(windows).astype(np.float32), logits=np.stack(logits).astype(np.float32),
                            **{"contacts_" + n: contacts[n] for n in lens})
    for n in lens:
        print(n, contacts[n].shape, contacts[n].dtype, contacts[n].sum(0))
    print("min |logit|", np.abs(np.stack(logits)).min())


if __name__ == "__main__":
    main()
