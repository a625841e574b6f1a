"""TEST INFRASTRUCTURE ONLY -- CPU checker of the contact classifier's labelled evaluation (`chd_k_contact_score`).

Restates in numpy what test.py:64-140 (val_full_video with labels) computes for one video from its window logits:
OpenPoseModel.loss summed, OpenPoseModel.accuracy for each predicted frame, and the count of the merged (voted) labels
against the label rows test.py rebuilds from the windows.  PINNED: checked against the counts and loss the reference's
own code produced (tests/golden/make_contact_eval_golden.py -> tests/golden/contact/contact_eval_golden.npz) in
tests/test_contact_eval_cpu.py.
"""
import numpy as np

from oracle.contact import vote


def fix_truth(truth, n_frames):
    """fix_data_len (real_video_dataset.py:165-191) for the contacts: (T,4) padded with the last row or trimmed to n_frames."""
    t = np.asarray(truth).reshape(-1, 4)
    if t.shape[0] >= n_frames:
        return t[:n_frames]
    return np.concatenate([t, np.repeat(t[-1:], n_frames - t.shape[0], axis=0)], axis=0)


def counts(pred, lab):
    """(tp, fp, fn, tn) of two boolean arrays."""
    return np.array([(pred & lab).sum(), (pred & ~lab).sum(), (~pred & lab).sum(), (~pred & ~lab).sum()], dtype=np.int64)


def score(logits, truth, thresh=0.5, window=9, pred=5):
    """logits (Wn,5,4) fp32 of one video padded to Fmax = Wn + 8 frames, truth (T,4) or None ->
    (loss_sum, conf_frames (5,4), conf_merged (4,)); zeros for a video without truth rows.
      loss_sum     sum of (1 - y) x - log_sigmoid(x), every term in fp32 (torch's binary_cross_entropy_with_logits), fp64 sum
      conf_frames  per predicted frame p: sigmoid(x) > thresh against truth row w + 2 + p of window w
      conf_merged  the 0.5 vote over all Fmax frames (before trimming) against truth row clamp(f, 2, Fmax - 3)"""
    x = np.asarray(logits, dtype=np.float32)
    Wn = x.shape[0]
    Fmax = Wn + window - 1
    if truth is None or np.asarray(truth).size == 0:
        return 0.0, np.zeros((pred, 4), dtype=np.int64), np.zeros(4, dtype=np.int64)
    t = fix_truth(truth, Fmax) != 0
    off = (window - pred) // 2
    y = np.stack([t[w + off:w + off + pred] for w in range(Wn)])                      # (Wn, 5, 4) label windows
    yf = y.astype(np.float32)
    one = np.float32(1)
    log_sig = np.minimum(x, np.float32(0)) - np.log1p(np.exp(-np.abs(x)))
    loss = float(np.sum(((one - yf) * x - log_sig).astype(np.float32), dtype=np.float64))
    p = (one / (one + np.exp(-x))) > np.float32(thresh)
    conf_frames = np.stack([counts(p[:, q], y[:, q]) for q in range(pred)])
    merged = vote(x, Fmax, window, pred) != 0                                        # (Fmax, 4), untrimmed
    rows = np.clip(np.arange(Fmax), off, Fmax - 1 - off)
    return loss, conf_frames, counts(merged, t[rows])
