"""Contact-net inference benchmark (BASELINE.json configs[2]: 100k 9-frame OpenPose-25 windows, 1 H100); reached as
`python bench.py --workload contact [--impl reference]`.  Prints one JSON line in bench.py's schema:

value : windows/s with the preprocessed keypoints already resident in HBM (`chd_contact_forward_device`)
e2e   : windows/s through the public host call `ContactNet.detect` (`chd_contact_detect`): raw OpenPose keypoints in
        page-locked host memory -> H2D -> preprocessing kernel -> windows / MLP / votes -> D2H of the int64 labels
--reference : the CPU arm -- the oracle restatement of the reference's dataset preprocessing + torch-CPU fp32 forward +
        vote aggregation on a bounded sample of the same videos, all host threads
--dump-outputs DIR : labels and logits of the last timed device-resident step as DIR/<name>.npy (float32)
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import numpy as np

V, F = 1000, 108                      # 1000 videos x 100 windows
CONFIG = {"workload": "contact-net inference: 100k 9-frame OpenPose-25 joint windows (%d synthetic videos x %d frames), 1 H100" % (V, F),
          "videos": V, "frames": F, "windows": V * (F - 8)}


def make_raw(n):
    from make_contact_golden import synth_keypoints
    rng = np.random.default_rng(0)
    base = [synth_keypoints(i, F) for i in range(8)]
    return [base[i % 8] + rng.normal(0, 0.5, base[0].shape) * np.array([1, 1, 0]) for i in range(n)]


def card():
    """Name, power limit and maximum SM clock of cuda:0, to state beside numbers measured in the same run."""
    import torch
    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "max_sm_clock_mhz": None}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        out["power_limit_w"], out["max_sm_clock_mhz"] = float(q[0]), float(q[1])
    except Exception as e:                                     # reported, not guessed
        out["query_error"] = repr(e)
    return out


def cpu_arm(raw, sd, threads):
    import torch
    from oracle import contact as oc
    torch.set_num_threads(threads)
    t0 = time.perf_counter()
    frames, lens = oc.preprocess_videos(raw)
    logits = oc.forward_torch(sd, oc.windows_from_frames(frames))
    labels = [oc.vote(logits[i], int(lens[i])) for i in range(len(raw))]
    return time.perf_counter() - t0, labels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reference", action="store_true")
    ap.add_argument("--cpu-videos", type=int, default=100)
    ap.add_argument("--dump-outputs", metavar="DIR")
    args = ap.parse_args()
    import torch
    from make_contact_golden import contact_weights
    sd = contact_weights(0)
    cores = os.cpu_count() or 1
    nwin = V * (F - 8)
    if args.reference:
        ns = args.cpu_videos
        raw = make_raw(ns)
        ts = [cpu_arm(raw, sd, cores)[0] for _ in range(max(1, args.steps))]
        v = ns * (F - 8) / float(np.mean(ts))
        print(json.dumps({"impl": "reference", "metric": "contact windows/s", "value": v, "unit": "windows/s", "n_gpus": 1, "steps": args.steps,
                          "warmup": args.warmup, "ms_per_step": 1e3 * float(np.mean(ts)), "higher_is_better": True, "scaling": "weak",
                          "vs_baseline": None, "dtype": "f32", "data": "synthetic", "config": CONFIG,
                          "cpu_baseline": {"value": v, "unit": "windows/s", "cores": cores, "kind": "port",
                                           "sample": "%d of the %d videos (%d windows) per step: numpy preprocessing + torch fp32 CPU forward + votes" % (ns, V, ns * (F - 8))},
                          "e2e": {"value": v, "unit": "windows/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}))
        return
    import chd
    raw = make_raw(V)
    cat, offs = chd.contact.concat_videos(raw)
    cat = torch.from_numpy(cat).pin_memory().numpy()            # page-locked host buffer for the e2e leg
    net = chd.contact.ContactNet(sd)
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device="cuda")   # 256 MiB > L2
    # ---- e2e through the public call ----
    for _ in range(args.warmup):
        labels, mabs = net.detect(None, cat=cat, offs=offs)
    l0 = net.launch_count()
    te = []
    for _ in range(args.steps):
        flush.zero_()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        labels, mabs = net.detect(None, cat=cat, offs=offs)
        te.append(time.perf_counter() - t0)
    launches = net.launch_count() - l0
    e2e = float(np.mean(te))
    # ---- device resident ----
    L = net.L
    frames, lens = net.preprocess(raw)
    fr, sl = torch.from_numpy(frames).cuda(), torch.from_numpy(lens).cuda()
    lab = torch.empty((V, F, 4), dtype=torch.int64, device="cuda")
    lg = torch.empty((nwin, 20), dtype=torch.float32, device="cuda")
    mn = torch.empty(1, dtype=torch.float32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    ts = []
    for i in range(args.warmup + args.steps):
        flush.zero_()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        L.chd_contact_forward_device(net.h, fr.data_ptr(), V, F, sl.data_ptr(), lab.data_ptr(), lg.data_ptr(), mn.data_ptr(), st)
        e1.record()
        torch.cuda.synchronize()
        if i >= args.warmup:
            ts.append(e0.elapsed_time(e1) * 1e-3)
    dev = float(np.mean(ts))
    lab_h = lab.cpu().numpy()
    assert all(np.array_equal(lab_h[i, :lens[i]], labels[i]) for i in range(V))
    # ---- bounded CPU sample (same videos) ----
    ns = args.cpu_videos
    cpu_t, ref_lab = cpu_arm(raw[:ns], sd, cores)
    agree = float(np.mean([np.array_equal(ref_lab[i], labels[i]) for i in range(ns)]))
    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        np.save(os.path.join(args.dump_outputs, "labels.npy"), lab_h.astype(np.float32))
        np.save(os.path.join(args.dump_outputs, "logits.npy"), lg.cpu().numpy())
    flops = 2 * 953984 * nwin
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    peak = sms * 128 * 2 * 1.98e9 / 1e12
    print(json.dumps({"metric": "contact windows/s", "value": nwin / dev, "unit": "windows/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
                      "ms_per_step": 1e3 * dev, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
                      "config": CONFIG,
                      "e2e": {"value": nwin / e2e, "unit": "windows/s", "h2d_bytes_per_step": int(cat.nbytes + offs.nbytes),
                              "d2h_bytes_per_step": int(sum(l.nbytes for l in labels)),
                              "includes": "H2D of the raw keypoints (page-locked), preprocessing kernel, windows + MLP + votes, D2H of the labels"},
                      "gpu_launches": int(launches),
                      "roofline": {"bound": "tensor", "kernel": "chd_k_contact_gemm", "achieved": flops / dev / 1e12, "peak": peak, "unit": "TFLOP/s",
                                   "frac": flops / dev / 1e12 / peak, "traffic": None,
                                   "note": "fp32 FFMA pipe (no tensor core: integer labels must match the reference's fp32 forward); peak = nominal SMs x 128 FFMA x 1.98 GHz (H100 SXM boost clock)"},
                      "cpu_baseline": {"value": ns * (F - 8) / cpu_t, "unit": "windows/s", "cores": cores, "kind": "port",
                                       "sample": "%d of the %d videos (%d windows): numpy preprocessing + torch fp32 CPU forward + votes, %.1f s" % (ns, V, ns * (F - 8), cpu_t)},
                      "labels_equal_frac_vs_cpu": agree, "min_abs_logit": mabs}))


if __name__ == "__main__":
    main()
