"""Generates the golden vectors of the contact classifier's labelled evaluation by running the REFERENCE's own code
(src/contact_learning of a checkout of the reference at $CHD_REFERENCE_DIR, default ../contact-human-dynamics next to
this repository: OpenPoseDataset, RealVideoDataset, OpenPoseModel, test.val_full_video) with the seeded weights
contact_weights(0) on
  * a synthetic tree from chd.synth.write_contact_dataset (2 characters x 10 motions x 2 views x 48 frames, seed 0:
    the test and val splits are not empty), read as test.py does without --real-data (overlap_test=True);
  * three real-video directories whose ground truth is longer than, shorter than, and missing relative to the keypoints.
The reference returns normalised confusion matrices only, so OpenPoseModel.accuracy and .loss are wrapped to record the
integer counts and the loss of every video.  The tree is not stored: the tests regenerate it from its seed.

    CHD_REFERENCE_DIR=/path/to/contact-human-dynamics python tests/golden/make_contact_eval_golden.py

Stubs and the np.int alias as in make_contact_golden.py.  Nothing from the reference is copied into the repo.
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_contact_golden import REF, ROOT, contact_weights, synth_keypoints, write_openpose_dir  # noqa: E402

sys.path.insert(0, ROOT)
TREE = dict(characters=2, motions=10, views=2, frames=48, seed=0)
REAL = {"vid_long": (50, 62), "vid_none": (61, None), "vid_short": (44, 30)}   # keypoint frames, truth rows


def stub_imports():
    import types
    for name in ["skimage", "skimage.io", "skimage.transform", "matplotlib", "matplotlib.pyplot", "matplotlib.animation",
                 "matplotlib.patheffects", "mpl_toolkits", "mpl_toolkits.mplot3d", "torchvision", "torchvision.transforms",
                 "torchvision.utils", "cv2"]:
        if name not in sys.modules:
            try:
                __import__(name)
            except Exception:
                sys.modules[name] = types.ModuleType(name)
    np.int = int


def truth_rows(seed, n):
    """Contact runs of 3..12 frames per column."""
    rng = np.random.default_rng(seed)
    out = np.zeros((n, 4), dtype=np.int64)
    for c in range(4):
        f, s = 0, int(rng.integers(0, 2))
        while f < n:
            L = int(rng.integers(3, 13))
            out[f:f + L, c] = s
            s, f = 1 - s, f + L
    return out


def run(ds, model, ref_test):
    """val_full_video on one dataset with OpenPoseModel.loss / .accuracy recorded per call; returns the logits of every
    window (V, Wn, 5, 4), the per-video records and what val_full_video returned."""
    import torch
    from torch.utils.data import DataLoader
    calls = []
    loss0, acc0 = model.loss, model.accuracy

    def loss(o, l):
        r = loss0(o, l)
        calls.append(("loss", float(torch.sum(r).item()), int(r.numel())))
        return r

    def accuracy(o, l, thresh=0.5, tgt_frame=None):
        r = acc0(o, l, thresh=thresh, tgt_frame=tgt_frame)
        calls.append(("acc", np.array(r, dtype=np.int64)))
        return r
    model.loss, model.accuracy = loss, accuracy
    loader = DataLoader(ds, batch_size=ds.get_num_test_windows_per_seq(), shuffle=False, num_workers=0)
    with torch.no_grad():
        logits = np.stack([model(b["joint2d"]).numpy() for b in loader])
        res = ref_test.val_full_video(loader, ds, model, torch.device("cpu"), 0.5, 5)
    model.loss, model.accuracy = loss0, acc0
    return logits, calls, res


def per_video(calls, labelled):
    """calls of val_full_video: per labelled video one loss, five per-frame and one merged accuracy call."""
    V = len(labelled)
    loss, count = np.zeros(V), np.zeros(V, dtype=np.int64)
    frames, merged = np.zeros((V, 5, 4), dtype=np.int64), np.zeros((V, 4), dtype=np.int64)
    i = 0
    for v in range(V):
        if not labelled[v]:
            continue
        assert calls[i][0] == "loss" and all(c[0] == "acc" for c in calls[i + 1:i + 7])
        loss[v], count[v] = calls[i][1], calls[i][2]
        frames[v] = np.stack([c[1] for c in calls[i + 1:i + 6]])
        merged[v] = calls[i + 6][1]
        i += 7
    assert i == len(calls)
    return loss, count, frames, merged


def main():
    stub_imports()
    import torch
    import chd
    os.chdir(REF)
    for p in ["contact_learning", ".", "utils", "optimize"]:
        sys.path.insert(0, os.path.join(REF, p))
    from models.openpose_only import OpenPoseModel
    from data.openpose_dataset import OpenPoseDataset
    from data.real_video_dataset import RealVideoDataset
    import test as ref_test

    model = OpenPoseModel(9, 13, 5, 3)
    model.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in contact_weights(0).items()})
    model.eval()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        # ---- synthetic tree ----
        root = os.path.join(tmp, "synth")
        chd.synth.write_contact_dataset(root, **TREE)
        names = {}
        for split in ("train", "test", "val"):
            ds = OpenPoseDataset(root, split=split, window_size=9, contact_size=5, load_img=False, overlap_test=True,
                                 use_confidence=True, joint_set="lower")
            names[split] = ["/".join(p.split("/")[-3:]) for p in ds.view_dirs]
        ds = OpenPoseDataset(root, split="test", window_size=9, contact_size=5, load_img=False, overlap_test=True,
                             use_confidence=True, joint_set="lower")
        logits, calls, (mean_loss, _, _) = run(ds, model, ref_test)
        loss, count, frames, merged = per_video(calls, [True] * len(ds.op_data))
        out.update({"synth_" + k: np.array(v) for k, v in names.items()})
        out.update(synth_median=np.float64(ds.normalization_info), synth_frames=np.stack(ds.op_data), synth_logits=logits.astype(np.float32),
                   synth_loss=loss, synth_count=count, synth_conf_frames=frames, synth_conf_merged=merged, synth_mean_loss=np.float64(mean_loss),
                   synth_tree=np.array([TREE[k] for k in ("characters", "motions", "views", "frames", "seed")]))
        # ---- real videos ----
        vids = sorted(REAL)
        data = os.path.join(tmp, "real")
        for i, n in enumerate(vids):
            F, T = REAL[n]
            kp = synth_keypoints(300 + i, F)
            write_openpose_dir(os.path.join(data, n, "openpose_result"), kp)
            if F > 45:                     # write_openpose_dir leaves frame 5 without detections: zeros when read
                kp[5] = 0.0
            out["real_raw_" + n] = kp
            if T is not None:
                t = truth_rows(400 + i, T)
                np.save(os.path.join(data, n, "foot_contacts.npy"), t)
                out["real_truth_" + n] = t
        ds = RealVideoDataset(data, split="test", window_size=9, contact_size=5, load_img=False, use_confidence=True, joint_set="lower")
        logits, calls, (mean_loss, _, _) = run(ds, model, ref_test)
        loss, count, frames, merged = per_video(calls, [REAL[n][1] is not None for n in vids])
        out.update(real_names=np.array(vids), real_logits=logits.astype(np.float32), real_loss=loss, real_count=count,
                   real_conf_frames=frames, real_conf_merged=merged, real_mean_loss=np.float64(mean_loss))
    np.savez_compressed(os.path.join(HERE, "contact", "contact_eval_golden.npz"), **out)
    for k in ("synth", "real"):
        print(k, "mean loss", out[k + "_mean_loss"], "per-frame", out[k + "_conf_frames"].sum(0).tolist(), "merged",
              out[k + "_conf_merged"].sum(0).tolist(), "min |logit|", float(np.abs(out[k + "_logits"]).min()))
    print("median", out["synth_median"], "test", list(out["synth_test"]))


if __name__ == "__main__":
    main()
