"""Cost of the contact classifier's labelled evaluation (`chd_k_contact_score`, `ContactNet.evaluate`) at the shape of
BASELINE.json configs[2]: 1000 videos x 108 frames (100k windows) with ground truth.  The videos are the walks of a
`chd.synth.write_contact_dataset` tree (16 training sequences of 108 frames, read by `read_synthetic_videos`), repeated
with pixel noise.  Prints one JSON line:

score_kernel_ms     : chd_k_contact_score alone (CUDA events around 50 launches after the forward)
device_resident     : windows/s of forward + vote + score and of forward + vote, alternated step by step after a
                      warm-up; median and (min, max) over --steps steps each
e2e                 : windows/s of ContactNet.evaluate from page-locked raw keypoints (upload, prep, forward, vote,
                      score, pack, download)
cpu_baseline        : the oracle arm (numpy preprocessing, torch fp32 CPU forward, numpy scoring) on --cpu-videos videos
gpu                 : card name, power limit and max SM clock, read in the same run

    python scripts/bench_contact_eval.py --steps 30 --warmup 5
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import numpy as np

from bench_contact import F, V, card


def make_videos(chd):
    with tempfile.TemporaryDirectory() as tmp:
        chd.synth.write_contact_dataset(tmp, 2, 10, 1, F, 0)
        s = chd.contact.read_synthetic_videos(tmp, "train").videos
    rng = np.random.default_rng(0)
    n = len(s.raw)
    raw = [s.raw[i % n] + rng.normal(0, 0.5, s.raw[0].shape) * np.array([1, 1, 0]) for i in range(V)]
    truth = [s.truth[i % n] for i in range(V)]
    return raw, truth, s.scale, s.norm


def cpu_arm(raw, truth, scale, norm, sd, threads):
    import torch
    from oracle import contact as oc
    from oracle.contact_eval import score
    torch.set_num_threads(threads)
    t0 = time.perf_counter()
    frames, _ = oc.preprocess_videos(raw, scale=scale, norm=norm)
    logits = oc.forward_torch(sd, oc.windows_from_frames(frames))
    res = [score(logits[i], truth[i]) for i in range(len(raw))]
    return time.perf_counter() - t0, res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--cpu-videos", type=int, default=50)
    args = ap.parse_args()
    import torch
    import chd
    from make_contact_golden import contact_weights
    sd = contact_weights(0)
    raw, truth, scale, norm = make_videos(chd)
    nwin = V * (F - 8)
    net = chd.contact.ContactNet(sd)
    L = net.L
    # ---- device resident: forward + vote (+ score) on preprocessed frames in HBM ----
    frames, lens = net.preprocess(raw, scale=scale, norm=norm)
    fr, sl = torch.from_numpy(frames).cuda(), torch.from_numpy(lens).cuda()
    lab = torch.empty((V, F, 4), dtype=torch.int64, device="cuda")
    lg = torch.empty((nwin, 20), dtype=torch.float32, device="cuda")
    mn = torch.empty(1, dtype=torch.float32, device="cuda")
    tr = torch.from_numpy(np.ascontiguousarray(np.concatenate(truth) != 0, dtype=np.int32)).cuda()
    toffs = torch.from_numpy(np.concatenate([[0], np.cumsum([t.shape[0] for t in truth])]).astype(np.int32)).cuda()
    loss = torch.empty(V, dtype=torch.float64, device="cuda")
    cf = torch.empty((V, 5, 4), dtype=torch.int64, device="cuda")
    cm = torch.empty((V, 4), dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def forward():
        rc = L.chd_contact_forward_device(net.h, fr.data_ptr(), V, F, sl.data_ptr(), lab.data_ptr(), lg.data_ptr(), mn.data_ptr(), st)
        assert rc == 0, rc

    def score():
        rc = L.chd_contact_score_device(net.h, lg.data_ptr(), V, F, tr.data_ptr(), toffs.data_ptr(), 0.5, loss.data_ptr(), cf.data_ptr(),
                                        cm.data_ptr(), st)
        assert rc == 0, rc

    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    legs = {"forward_vote": forward, "forward_vote_score": lambda: (forward(), score())}
    ms = {k: [] for k in legs}
    for i in range(args.warmup + args.steps):
        for k, fn in legs.items():
            t = timed(fn)
            if i >= args.warmup:
                ms[k].append(t)
    forward()
    reps = 50
    score_ms = timed(lambda: [score() for _ in range(reps)]) / reps
    dev = {"forward_vote_score_ms": ms["forward_vote_score"], "forward_vote_ms": ms["forward_vote"]}
    # ---- e2e through the public call from page-locked raw keypoints ----
    cat, offs = chd.contact.concat_videos(raw)
    cat = torch.from_numpy(cat).pin_memory().numpy()
    for _ in range(args.warmup):
        res = net.evaluate(None, truth, scale, norm, cat=cat, offs=offs)
    te = []
    for _ in range(args.steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = net.evaluate(None, truth, scale, norm, cat=cat, offs=offs)
        te.append(time.perf_counter() - t0)
    # the device-resident score equals the public call's
    assert np.array_equal(cf.cpu().numpy(), res["conf_frames"]) and np.array_equal(cm.cpu().numpy(), res["conf_merged"])
    # ---- CPU arm on a bounded sample ----
    cores = os.cpu_count() or 1
    ns = args.cpu_videos
    cpu_t, cpu_res = cpu_arm(raw[:ns], truth[:ns], scale, norm, sd, cores)
    agree = float(np.mean([np.array_equal(cpu_res[i][1], res["conf_frames"][i]) and np.array_equal(cpu_res[i][2], res["conf_merged"][i])
                           for i in range(ns)]))

    def rate(xs):
        xs = np.asarray(xs)
        return {"median": nwin / (np.median(xs) * 1e-3), "min": nwin / (xs.max() * 1e-3), "max": nwin / (xs.min() * 1e-3),
                "median_ms": float(np.median(xs))}
    print(json.dumps({"metric": "contact evaluation windows/s", "config": {"videos": V, "frames": F, "windows": nwin, "steps": args.steps,
                                                                           "warmup": args.warmup},
                      "score_kernel_ms": score_ms,
                      "device_resident": {"forward_vote_score": rate(dev["forward_vote_score_ms"]), "forward_vote": rate(dev["forward_vote_ms"]),
                                          "unit": "windows/s"},
                      "e2e": {"value": nwin / float(np.median(te)), "unit": "windows/s", "median_ms": 1e3 * float(np.median(te)),
                              "min_ms": 1e3 * float(np.min(te)), "max_ms": 1e3 * float(np.max(te))},
                      "mean_loss": res["mean_loss"], "min_abs_logit": res["min_abs_logit"],
                      "cpu_baseline": {"value": ns * (F - 8) / cpu_t, "unit": "windows/s", "threads": cores, "videos": ns, "seconds": cpu_t,
                                       "counts_equal_frac_vs_gpu": agree},
                      "gpu": card()}))


if __name__ == "__main__":
    main()
