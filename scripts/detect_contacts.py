#!/usr/bin/env python
"""Drop-in for the reference's `python contact_learning/test.py --data D --out O --weights-path W --full-video
[--save-contacts] [--real-data]` (scripts/run_detect_contacts.py:51-58, README "Training and Testing Contact Detection
Network on Synthetic Data").

Data layouts:
* real videos, D/<video>/openpose_result/*_keypoints.json (+ D/<video>/foot_contacts.npy when the truth is known): every
  video's labels go to O/contact_results/<video>/foot_contacts.npy (int64, F x 4, columns L heel, L toe, R heel, R toe),
  with or without --save-contacts.  With `--copy-into-data` it also performs run_detect_contacts.py:65-69 (copy into
  each video directory).  This layout is used with --real-data, and also without it: the reference then reads D as the
  synthetic dataset and fails on this input, so existing callers that leave the flag out see no change.
* the synthetic dataset, D/<character>/<motion>/{foot_contacts.npy, view<k>/*.png, keypoints_view<k>/}: its test split
  (OpenPoseDataset, overlap_test=True) is evaluated.  --save-contacts writes
  O/contact_results/<character>/<motion>/view<k>/foot_contacts.npy with all frames; the reference raises
  KeyError: 'seq_len' there, since its synthetic items carry no sequence length.

When any video has ground truth the reference's result block is printed (TEST RESULTS, Mean Loss, the metrics of each
predicted frame, FULL VIDEO MERGED RESULTS) and the same numbers, with the raw (tp, fp, fn, tn) counts, go to
O/test_metrics.json; the reference draws confusion-matrix PNGs instead.  --classify-thresh sets the threshold of the
per-frame counts, as in test.py; the merged labels always use the 0.5 vote.  --viz is accepted and ignored."""
import argparse
import json
import os
import shutil
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def parse_args(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--data", required=True)
    ap.add_argument("--out", required=True)
    ap.add_argument("--weights-path", "--weights", dest="weights", required=True)
    ap.add_argument("--full-video", action="store_true")
    ap.add_argument("--save-contacts", action="store_true")
    ap.add_argument("--real-data", action="store_true")
    ap.add_argument("--viz", action="store_true")
    ap.add_argument("--classify-thresh", type=float, default=0.5)
    ap.add_argument("--copy-into-data", action="store_true")
    ap.add_argument("--precision", choices=["fp32", "tf32x3"], default="fp32",
                    help="fp32: labels match the reference's fp32 forward; tf32x3: the large layers on the tensor core "
                         "with split TF32 operands")
    return ap.parse_args(argv)


def metrics_entry(counts):
    """utils.py:73-96 calculate_metrics through chd.train.metrics, with the raw counts and the normalised matrix."""
    import chd
    import numpy as np
    c = np.asarray(counts, dtype=np.int64)
    acc, p, r, f1 = chd.train.metrics(c)
    return {"accuracy": acc, "precision": p, "recall": r, "f1": f1, "counts": dict(zip(("tp", "fp", "fn", "tn"), (int(v) for v in c))),
            "confusion_matrix": (c.reshape(2, 2) / max(int(c.sum()), 1)).tolist()}


def print_metrics(m):
    """utils.py:98-108."""
    cm = m["confusion_matrix"]
    print("Accuracy: %.3f" % m["accuracy"])
    print("Precision: %.3f" % m["precision"])
    print("Recall: %.3f" % m["recall"])
    print("F1 Score: %.3f" % m["f1"])
    print("Confusion Matrix:")
    print("                 + Actual -   ")
    print(" Predicted  + | %.3f  %.3f |" % (cm[0][0], cm[0][1]))
    print("            - | %.3f  %.3f |" % (cm[1][0], cm[1][1]))


def report(res, names, args):
    """test.py:301-312 on stdout; the same numbers and the per-video counts as a dict (test_metrics.json)."""
    frames = [metrics_entry(c) for c in res["frames_total"]]
    merged = metrics_entry(res["merged_total"])
    print("==================== TEST RESULTS ===========================================")
    print("Mean Loss: %0.3f" % res["mean_loss"])
    for i, m in enumerate(frames):
        print("----- Pred Frame " + str(i) + " ------")
        print_metrics(m)
    print("=======================================================")
    print("============== FULL VIDEO MERGED RESULTS ======================")
    print_metrics(merged)
    print("===============================================================")
    per_video = [{"name": n, "loss_sum": float(res["loss_sum"][i]), "conf_frames": res["conf_frames"][i].tolist(),
                  "conf_merged": res["conf_merged"][i].tolist()} for i, n in enumerate(names)]
    return {"mean_loss": res["mean_loss"], "loss_sum": float(res["loss_sum"].sum()), "loss_count": res["loss_count"],
            "videos": len(names), "labelled_videos": res["labelled"], "windows_per_video": res["windows"],
            "classify_thresh": args.classify_thresh, "precision": args.precision, "pred_frames": frames, "merged": merged,
            "per_video": per_video}


def main(argv=None):
    args = parse_args(argv)
    import chd
    layout, vids = chd.contact.read_videos(args.data, args.real_data)
    sd = chd.contact.load_weights(args.weights)
    net = chd.contact.ContactNet(sd, precision=args.precision)
    if layout == "real" and all(t is None for t in vids.truth):
        labels, _ = net.detect(vids.raw)
    else:
        res = net.evaluate(vids.raw, vids.truth, vids.scale, vids.norm, classify_thresh=args.classify_thresh)
        labels = res["labels"]
        if res["labelled"]:
            os.makedirs(args.out, exist_ok=True)
            with open(os.path.join(args.out, "test_metrics.json"), "w") as fh:
                json.dump(report(res, vids.names, args), fh, indent=1)
    if layout == "real" or args.save_contacts:
        for w in chd.contact.save_contacts(args.out, vids.names, labels):
            print("wrote", w)
            if args.copy_into_data and layout == "real":
                shutil.copyfile(w, os.path.join(args.data, os.path.basename(os.path.dirname(w)), "foot_contacts.npy"))


if __name__ == "__main__":
    main()
