"""Contact-net inference in both numerical modes on the workload of scripts/bench_contact.py (100k 9-frame OpenPose-25
windows: 1000 synthetic videos x 108 frames, contact_weights(0)).  The two modes run in one process, alternating step
by step after warm-up, with a 256 MiB L2 flush before each step:

device : `chd_contact_forward_device` with the preprocessed keypoints resident in HBM, timed with CUDA events
e2e    : `ContactNet.detect` from page-locked raw keypoints (H2D, preprocessing, network, votes, D2H of the labels),
         host clock after a synchronise

Prints one JSON line: card and power limit, windows/s, ms per step (mean, min, max), counted TFLOP/s
(2 x 953,984 flop per window) per mode, the fast mode's tensor-core work (three TF32 products on the 1.90 MF per
window of the three large layers), max |logit difference|, the fraction of videos with identical labels, min |logit|,
and the smallest |fp32 logit| of each video whose labels differ.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import numpy as np

from bench_contact import CONFIG, F, V, make_raw

FLOP_PER_WINDOW = 2 * 953984                                   # all five layers, as counted by bench_contact.py
TC_MAC_PER_WINDOW = 352 * 1024 + 1024 * 512 + 512 * 128        # the three tensor-core layers (K of layer 0 padded to 352)
MODES = ("fp32", "tf32x3")


def card():
    import torch
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "max_sm_clock_mhz": None}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        out["power_limit_w"], out["max_sm_clock_mhz"] = float(q[0]), float(q[1])
    except Exception as e:                                     # reported, not guessed
        out["query_error"] = repr(e)
    return out


def stats(ts):
    ts = np.asarray(ts)
    return {"ms_mean": 1e3 * float(ts.mean()), "ms_min": 1e3 * float(ts.min()), "ms_max": 1e3 * float(ts.max()),
            "ms_std": 1e3 * float(ts.std())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    import chd
    from make_contact_golden import contact_weights
    if not torch.cuda.is_available():
        raise SystemExit("bench_contact_precision: no CUDA device")
    sd = contact_weights(0)
    nwin = V * (F - 8)
    raw = make_raw(V)
    cat, offs = chd.contact.concat_videos(raw)
    cat = torch.from_numpy(cat).pin_memory().numpy()
    nets = {m: chd.contact.ContactNet(sd, precision=m) for m in MODES}
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device="cuda")   # 256 MiB > L2
    frames, lens = nets["fp32"].preprocess(raw)
    fr, sl = torch.from_numpy(frames).cuda(), torch.from_numpy(lens).cuda()
    out = {m: (torch.empty((V, F, 4), dtype=torch.int64, device="cuda"), torch.empty((nwin, 20), dtype=torch.float32, device="cuda"),
               torch.empty(1, dtype=torch.float32, device="cuda")) for m in MODES}
    st = torch.cuda.current_stream().cuda_stream
    fwd = nets["fp32"].L.chd_contact_forward_device

    def device_step(m):
        lab, lg, mn = out[m]
        flush.zero_()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rc = fwd(nets[m].h, fr.data_ptr(), V, F, sl.data_ptr(), lab.data_ptr(), lg.data_ptr(), mn.data_ptr(), st)
        e1.record()
        torch.cuda.synchronize()
        assert rc == 0, rc
        return e0.elapsed_time(e1) * 1e-3

    def e2e_step(m):
        flush.zero_()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        labels, _ = nets[m].detect(None, cat=cat, offs=offs)
        return time.perf_counter() - t0, labels

    dev = {m: [] for m in MODES}
    e2e = {m: [] for m in MODES}
    det = {}
    for i in range(args.warmup + args.steps):
        for m in (MODES if i % 2 == 0 else MODES[::-1]):        # alternate which mode goes first
            t = device_step(m)
            if i >= args.warmup:
                dev[m].append(t)
    for i in range(args.warmup + args.steps):
        for m in (MODES if i % 2 == 0 else MODES[::-1]):
            t, det[m] = e2e_step(m)
            if i >= args.warmup:
                e2e[m].append(t)
    lab = {m: out[m][0].cpu().numpy() for m in MODES}
    lg = {m: out[m][1].cpu().numpy() for m in MODES}
    for m in MODES:                                             # detect and the device-resident call agree in each mode
        assert all(np.array_equal(lab[m][i, :lens[i]], det[m][i]) for i in range(V)), m
    res = {"workload": CONFIG["workload"], "windows": nwin, "steps": args.steps, "warmup": args.warmup, "card": card(), "modes": {}}
    for m in MODES:
        td, te = float(np.mean(dev[m])), float(np.mean(e2e[m]))
        res["modes"][m] = {"device": dict(stats(dev[m]), windows_per_s=nwin / td, tflops_counted=FLOP_PER_WINDOW * nwin / td / 1e12),
                           "e2e": dict(stats(e2e[m]), windows_per_s=nwin / te),
                           "min_abs_logit": float(np.abs(lg[m]).min())}
    ttc = float(np.mean(dev["tf32x3"]))
    tc_flop = 3 * 2 * TC_MAC_PER_WINDOW * nwin
    res["tf32x3_tensor_core"] = {"gflop": tc_flop / 1e9, "tflops": tc_flop / ttc / 1e12,
                                 "note": "three TF32 products (lo*hi, hi*lo, hi*hi) on the 352-1024-512-128 layers"}
    res["speedup_device"] = float(np.mean(dev["fp32"])) / ttc
    res["speedup_e2e"] = float(np.mean(e2e["fp32"])) / float(np.mean(e2e["tf32x3"]))
    res["max_abs_dlogit"] = float(np.abs(lg["tf32x3"] - lg["fp32"]).max())
    differ = [i for i in range(V) if not np.array_equal(lab["tf32x3"][i], lab["fp32"][i])]
    res["labels_equal_video_frac"] = 1.0 - len(differ) / V
    # every video whose labels differ: the smallest |fp32 logit| of that video (a flip needs a logit near zero)
    res["differing_videos_min_abs_logit"] = [float(np.abs(lg["fp32"].reshape(V, F - 8, 20)[i]).min()) for i in differ]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
