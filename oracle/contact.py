"""TEST INFRASTRUCTURE ONLY -- CPU oracle of the contact-classifier path.

Restates, in numpy / torch fp32, the dataset preprocessing of real_video_dataset.py:132-163 /
openpose_dataset.py:49-121 (the checker of the product's `chd_k_contact_prep` kernel), the window construction of real_video_dataset.py:206-276, the layer list of
models/openpose_only.py:29-44 (eval mode) and the vote aggregation of test.py:88-122.  PINNED: checked against the
golden vectors produced by the reference's own code (tests/golden/make_contact_golden.py ->
tests/golden/contact/contact_golden.npz) in tests/test_contact_cpu.py.
"""
import numpy as np

LOWER = [8, 9, 10, 11, 12, 13, 14, 19, 20, 21, 22, 23, 24]   # openpose_dataset.py:38
LIN_IDS, BN_IDS = [0, 3, 6, 10, 13], [1, 4, 7, 11]


TRAIN_DIM = (1280, 720)                      # real_video_dataset.py:17
TRAIN_NORMALIZATION = 200.4160302695367      # real_video_dataset.py:18


def interpolate_low_confidence(seq, thresh=0.2):
    """process_openpose_data (openpose_dataset.py:49-111) for one (F,J,3) sequence, in place on xy: per joint, leading /
    trailing low-confidence runs take the nearest confident frame, interior runs are blended between the confident
    frames on either side with a weight that is accumulated step by step (the reference's rounding)."""
    F, J = seq.shape[:2]
    low = seq[:, :, 2] < thresh
    for j in range(J):
        runs, t = [], 0
        while t < F:                       # maximal runs [a, b) of low-confidence frames
            if low[t, j]:
                b = t
                while b < F and low[b, j]:
                    b += 1
                runs.append((t, b))
                t = b
            else:
                t += 1
        for a, b in runs:
            if a == 0 and b == F:
                continue
            if a == 0:
                seq[:b, j, :2] = seq[b, j, :2]
            elif b == F:
                seq[a - 1:, j, :2] = seq[a - 1, j, :2]
            else:
                left, right = seq[a - 1, j, :2].copy(), seq[b, j, :2].copy()
                step = 1.0 / (b - (a - 1))
                w = step
                for t in range(a, b):
                    seq[t, j, :2] = (1.0 - w) * left + w * right
                    w += step
    return seq


def preprocess_videos(raw, dimensions=(1920, 1080), scale=None, norm=TRAIN_NORMALIZATION):
    """RealVideoDataset.__init__ (real_video_dataset.py:132-163): pad every video to the longest by repeating the last
    frame, scale xy by `scale` (default 1280/width), interpolate low-confidence joints, divide xy by `norm` (default the
    training normalisation; the synthetic dataset passes scale 1 and its median).
    Returns (frames (V,Fmax,25,3) fp64, seq_lens (V,) int32)."""
    seq_lens = np.array([r.shape[0] for r in raw], dtype=np.int32)
    Fmax = int(seq_lens.max())
    out = np.zeros((len(raw), Fmax, 25, 3))
    scale = float(TRAIN_DIM[0]) / dimensions[0] if scale is None else scale
    for i, r in enumerate(raw):
        a = np.array(r, dtype=np.float64)
        if a.shape[0] < Fmax:
            a = np.concatenate([a, np.repeat(a[-1:], Fmax - a.shape[0], axis=0)], axis=0)
        a[:, :, :2] *= scale
        a = interpolate_low_confidence(a, 0.2)
        a[:, :, :2] /= norm
        out[i] = a
    return out, seq_lens


def windows_from_frames(frames, window=9):
    """frames (V,Fmax,25,3) fp64 -> (V, Wn, 9, 13, 3) fp32, root (joint 8) of the centre frame subtracted from every
    xy and then restored on the centre frame itself (real_video_dataset.py:244-252)."""
    V, Fmax = frames.shape[:2]
    Wn = Fmax - (window - 1)
    out = np.zeros((V, Wn, window, len(LOWER), 3), dtype=np.float32)
    for v in range(V):
        for w in range(Wn):
            cur = frames[v, w:w + window].copy()
            root = cur[window // 2, 8, :2].copy().reshape((1, 1, 2))
            cur[:, :, :2] -= root
            cur[window // 2, 8, :2] = root
            out[v, w] = cur[:, LOWER, :].astype(np.float32)
    return out


def forward_torch(sd, windows):
    """windows (..., 9, 13, 3) fp32 -> logits (..., 5, 4); the reference's nn.Sequential in eval mode, torch CPU fp32."""
    import torch
    import torch.nn as nn
    model = nn.Sequential(nn.Linear(351, 1024), nn.BatchNorm1d(1024), nn.ReLU(), nn.Linear(1024, 512), nn.BatchNorm1d(512),
                          nn.ReLU(), nn.Linear(512, 128), nn.BatchNorm1d(128), nn.ReLU(), nn.Dropout(p=0.3),
                          nn.Linear(128, 32), nn.BatchNorm1d(32), nn.ReLU(), nn.Linear(32, 20))
    model.load_state_dict({k[len("model."):]: torch.from_numpy(np.asarray(v)) for k, v in sd.items()})
    model.eval()
    x = torch.from_numpy(np.ascontiguousarray(windows, dtype=np.float32)).reshape(-1, 351)
    with torch.no_grad():
        y = model(x).numpy()
    return y.reshape(windows.shape[:-3] + (5, 4))


def vote(logits, seq_len, window=9, pred=5):
    """logits (Wn,5,4) of one (padded) video -> int64 labels (seq_len,4): sigmoid>0.5, votes over the 5 overlapping
    predictions, thresholds [1,1,2,2,3,...,3,2,2,1,1], two copies padded on each side, trimmed (test.py:88-152)."""
    import torch
    p = (torch.sigmoid(torch.from_numpy(np.ascontiguousarray(logits, dtype=np.float32))) > 0.5).numpy()
    Wn = p.shape[0]
    agg = np.zeros((Wn + 2 * (pred // 2), 4))
    for w in range(Wn):
        agg[w:w + pred] += p[w]
    th = np.ones(agg.shape[0]) * ((pred + 1) / 2)
    for e in range(pred - 1):
        th[e] = e // 2 + 1
        th[-1 - e] = e // 2 + 1
    lab = (agg >= th.reshape((-1, 1))).astype(np.int64)
    off = (window - pred) // 2
    lab = np.concatenate([np.repeat(lab[:1], off, axis=0), lab, np.repeat(lab[-1:], off, axis=0)], axis=0)
    return lab[:seq_len]
