"""Host side of the foot-contact classifier path (reference: scripts/run_detect_contacts.py ->
src/contact_learning/test.py --full-video --save-contacts --real-data).

Keypoint loading (JSON) happens on the host; the dataset preprocessing (padding, scaling, low-confidence
interpolation, normalisation: real_video_dataset.py:132-163, openpose_dataset.py:49-121), window construction, the MLP
and the vote aggregation run in hand-written CUDA behind `chd_contact_*` (include/chd.h).  No CPU fallback.
With ground truth (test.py --full-video on labelled videos or on the synthetic dataset's test split) `ContactNet.evaluate`
also scores the windows on the device (`chd_contact_detect` with truth); `read_real_videos` / `read_synthetic_videos`
read the two dataset layouts.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, List, NamedTuple, Optional, Sequence

import numpy as np

from .phys import load_lib

TRAIN_DIM = (1280, 720)                      # real_video_dataset.py:17
TRAIN_NORMALIZATION = 200.4160302695367      # real_video_dataset.py:18
WINDOW, PRED = 9, 5
LIN_IDS, BN_IDS = [0, 3, 6, 10, 13], [1, 4, 7, 11]
DIMS = [351, 1024, 512, 128, 32, 20]


def video_scale(dimensions=(1920, 1080)) -> float:
    """xy factor of real videos, TRAIN_DIM[0] / dimensions[0] (real_video_dataset.py:149)."""
    return float(TRAIN_DIM[0]) / dimensions[0]


def load_keypoint_files(files: Sequence[str], num_joints: int = 25, threads: int = 0) -> np.ndarray:
    """Many OpenPose `*_keypoints.json` files -> (len(files), J, 3) fp64 through the native threaded reader
    (`chd_openpose_load`, csrc/chd_openpose.cpp); bit-identical to openpose_utils.py:48-66 applied per file."""
    L = load_lib()
    out = np.empty((len(files), num_joints, 3), dtype=np.float64)
    arr = (C.c_char_p * len(files))(*[os.fsencode(f) for f in files])
    rc = L.chd_openpose_load(arr, len(files), num_joints, out.ctypes.data_as(C.c_void_p), threads)
    if rc:
        raise RuntimeError("chd_openpose_load failed: %d (-2 unreadable file, -3 malformed keypoint file)" % rc)
    return out


def load_keypoint_file(path: str, num_joints: int = 25) -> np.ndarray:
    """openpose_utils.py:48-66: first person's pose_keypoints_2d as (J,3); zeros if nobody was detected."""
    return load_keypoint_files([path], num_joints)[0]


def keypoint_files(path: str) -> List[str]:
    """openpose_utils.py:72: the *.json of a directory in sorted order."""
    return sorted(os.path.join(path, f) for f in os.listdir(path) if f.split(".")[-1] == "json")


def load_keypoint_dir(path: str) -> np.ndarray:
    """openpose_utils.py:68-76: all *.json of a directory in sorted order -> (F,25,3)."""
    return load_keypoint_files(keypoint_files(path))


def load_keypoint_dirs(paths: Sequence[str], threads: int = 0) -> List[np.ndarray]:
    """Several videos at once: one pass of the threaded reader over all files of all directories."""
    lists = [keypoint_files(p) for p in paths]
    flat = load_keypoint_files([f for l in lists for f in l], threads=threads)
    out, o = [], 0
    for l in lists:
        out.append(flat[o:o + len(l)])
        o += len(l)
    return out


def concat_videos(raw: Sequence[np.ndarray]):
    """list of (F_i,25,3) keypoint arrays -> (sum F, 25, 3) fp64 + (V+1,) int32 frame offsets (what chd_contact_* take)."""
    offs = np.zeros(len(raw) + 1, dtype=np.int32)
    offs[1:] = np.cumsum([r.shape[0] for r in raw])
    return np.ascontiguousarray(np.concatenate([np.asarray(r, dtype=np.float64) for r in raw], axis=0)), offs


def pack_state_dict(sd: Dict[str, np.ndarray]):
    """Flattens a reference state_dict (numpy values) into the three arrays chd_contact_create takes."""
    w = np.concatenate([np.asarray(sd["model.%d.weight" % i], dtype=np.float32).reshape(-1) for i in LIN_IDS])
    b = np.concatenate([np.asarray(sd["model.%d.bias" % i], dtype=np.float32).reshape(-1) for i in LIN_IDS])
    bn = np.concatenate([np.concatenate([np.asarray(sd["model.%d.%s" % (i, k)], dtype=np.float32).reshape(-1)
                                         for k in ("weight", "bias", "running_mean", "running_var")]) for i in BN_IDS])
    return np.ascontiguousarray(w), np.ascontiguousarray(b), np.ascontiguousarray(bn)


def load_weights(path: str) -> Dict[str, np.ndarray]:
    """A reference `.pth` state_dict (torch.load) or an `.npz` with the same keys."""
    if path.endswith(".npz"):
        return dict(np.load(path))
    import torch
    sd = torch.load(path, map_location="cpu")
    return {k: v.numpy() for k, v in sd.items()}


PRECISIONS = {"fp32": 0, "tf32x3": 1}       # CHD_CONTACT_FP32, CHD_CONTACT_TF32X3 (include/chd.h)


def precision_code(precision: str) -> int:
    if precision not in PRECISIONS:
        raise ValueError("unknown contact precision %r: expected one of %s" % (precision, ", ".join(sorted(PRECISIONS))))
    return PRECISIONS[precision]


class ContactNet:
    """The classifier on one GPU.  `precision="fp32"` (default) is the FFMA path whose labels match the reference's
    fp32 forward; `"tf32x3"` runs the three large layers on the tensor core with split TF32 operands
    (`chd_contact_set_precision`), logits within a few 1e-5 of the fp32 mode."""

    def __init__(self, state_dict: Dict[str, np.ndarray], device: int = -1, bn_eps: float = 1e-5, precision: str = "fp32"):
        code = precision_code(precision)
        self.L = L = load_lib()
        w, b, bn = pack_state_dict(state_dict)
        assert w.size == sum(i * o for i, o in zip(DIMS[:-1], DIMS[1:])) and b.size == sum(DIMS[1:])
        h = C.c_void_p()
        rc = L.chd_contact_create(w.ctypes.data, b.ctypes.data, bn.ctypes.data, C.c_float(bn_eps), device, C.byref(h))
        if rc != 0:
            raise RuntimeError("chd_contact_create failed with code %d (no CUDA device? no CPU fallback exists)" % rc)
        self.h = h
        self.precision = "fp32"
        if code != PRECISIONS["fp32"]:
            self.set_precision(precision)

    def set_precision(self, precision: str):
        """Numerical mode of every later forward / detect call: "fp32" or "tf32x3"."""
        rc = self.L.chd_contact_set_precision(self.h, precision_code(precision))
        if rc != 0:
            raise RuntimeError("chd_contact_set_precision failed with code %d" % rc)
        self.precision = precision

    def close(self):
        if getattr(self, "h", None):
            self.L.chd_contact_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def forward(self, frames: np.ndarray, seq_lens: np.ndarray, want_logits: bool = False):
        """frames (V,Fmax,25,3) preprocessed fp64 -> labels (V,Fmax,4) int64 [, logits (V,Fmax-8,5,4)], min|logit|."""
        frames = np.ascontiguousarray(frames, dtype=np.float64)
        seq_lens = np.ascontiguousarray(seq_lens, dtype=np.int32)
        V, Fmax = frames.shape[:2]
        labels = np.zeros((V, Fmax, 4), dtype=np.int64)
        logits = np.zeros((V, Fmax - (WINDOW - 1), PRED, 4), dtype=np.float32) if want_logits else None
        mabs = np.zeros(1, dtype=np.float32)
        rc = self.L.chd_contact_forward(self.h, frames.ctypes.data, V, Fmax, seq_lens.ctypes.data, labels.ctypes.data,
                                        logits.ctypes.data if want_logits else None, mabs.ctypes.data)
        if rc != 0:
            raise RuntimeError("chd_contact_forward failed with code %d" % rc)
        return (labels, logits, float(mabs[0])) if want_logits else (labels, float(mabs[0]))

    def preprocess(self, raw: Sequence[np.ndarray], dimensions=(1920, 1080), scale: Optional[float] = None, norm: float = TRAIN_NORMALIZATION):
        """RealVideoDataset.__init__ on the device (`chd_contact_preprocess`): list of raw (F_i,25,3) keypoints ->
        (frames (V,Fmax,25,3) fp64, seq_lens (V,) int32), bit identical to the reference's numpy result.  `scale`
        (default 1280 / dimensions[0]) and `norm` are the dataset's constants; `SyntheticVideos` carries its own."""
        cat, offs = concat_videos(raw)
        V, Fmax = len(raw), int(np.diff(offs).max())
        frames = np.zeros((V, Fmax, 25, 3))
        lens = np.zeros(V, dtype=np.int32)
        scale = video_scale(dimensions) if scale is None else scale
        rc = self.L.chd_contact_preprocess(self.h, cat.ctypes.data, offs.ctypes.data, V, float(scale), float(norm), frames.ctypes.data,
                                           lens.ctypes.data)
        if rc != 0:
            raise RuntimeError("chd_contact_preprocess failed with code %d" % rc)
        return frames, lens

    def _detect(self, raw, cat, offs, scale, norm, truth=None, classify_thresh=0.5):
        """One `chd_contact_detect` call on `raw` or the concatenated `cat` / `offs` -> (labels per video, min |logit|, offs,
        truth offsets, (loss_sum, conf_frames, conf_merged)); without `truth` nothing is scored and those are None."""
        if cat is None:
            cat, offs = concat_videos(raw)
        V = len(offs) - 1
        lab = np.zeros((int(offs[-1]), 4), dtype=np.int64)
        mabs = np.zeros(1, dtype=np.float32)
        tcat, toffs, scores = None, None, (None,) * 3
        if truth is not None:
            if len(truth) != V:
                raise ValueError("evaluate: %d videos but %d truth entries" % (V, len(truth)))
            rows = [np.zeros((0, 4), dtype=np.int32) if t is None else np.asarray(t).reshape(-1, 4) for t in truth]
            toffs = np.zeros(V + 1, dtype=np.int32)
            toffs[1:] = np.cumsum([r.shape[0] for r in rows])
            tcat = np.ascontiguousarray(np.concatenate(rows, axis=0) != 0, dtype=np.int32) if toffs[-1] else np.zeros((1, 4), dtype=np.int32)
            scores = (np.zeros(V, dtype=np.float64), np.zeros((V, PRED, 4), dtype=np.int64), np.zeros((V, 4), dtype=np.int64))
        ptr = lambda a: None if a is None else a.ctypes.data
        rc = self.L.chd_contact_detect(self.h, cat.ctypes.data, offs.ctypes.data, V, float(scale), float(norm), ptr(tcat), ptr(toffs),
                                       C.c_float(classify_thresh), lab.ctypes.data, *map(ptr, scores), mabs.ctypes.data)
        if rc != 0:
            raise RuntimeError("chd_contact_detect failed with code %d" % rc)
        return [lab[offs[i]:offs[i + 1]] for i in range(V)], float(mabs[0]), offs, toffs, scores

    def detect(self, raw: Sequence[np.ndarray], dimensions=(1920, 1080), cat=None, offs=None):
        """raw keypoints -> list of (F_i,4) int64 foot-contact labels (`chd_contact_detect`: preprocessing, windows,
        network, votes on the device; one upload, one download).  `cat` / `offs` may carry a pre-concatenated (e.g.
        page-locked) buffer."""
        return self._detect(raw, cat, offs, video_scale(dimensions), TRAIN_NORMALIZATION)[:2]

    def evaluate(self, raw: Sequence[np.ndarray], truth: Sequence[Optional[np.ndarray]], scale: float, norm: float,
                 classify_thresh: float = 0.5, cat=None, offs=None) -> Dict:
        """test.py --full-video with ground truth (`chd_contact_detect`: preprocessing with `scale` / `norm`, windows,
        network, votes and scoring on the device; one upload, one download).  truth[i]: (T_i,4) contacts of video i (any
        length: padded with the last row or trimmed to the longest video, as fix_data_len does) or None.  Returns a dict:
          labels       list of (F_i,4) int64, what `detect` returns
          loss_sum     (V,) sum of the BCE-with-logits terms of every window of a labelled video
          conf_frames  (V,5,4) (tp, fp, fn, tn) of each predicted frame, sigmoid(x) > classify_thresh
          conf_merged  (V,4) (tp, fp, fn, tn) of the 0.5-vote labels over all frames of the padded video
          frames_total (5,4), merged_total (4,): the sums over the videos
          labelled, windows, loss_count: labelled videos, windows per video, terms in the mean loss
          mean_loss    loss_sum.sum() / loss_count (test.py:84-85, 214), None without labelled videos
          min_abs_logit"""
        labels, mabs, offs, toffs, (loss, cf, cm) = self._detect(raw, cat, offs, scale, norm, truth, classify_thresh)
        windows = int(np.diff(offs).max()) - (WINDOW - 1)
        labelled = int((np.diff(toffs) > 0).sum())
        count = PRED * 4 * windows * labelled
        return dict(labels=labels, loss_sum=loss, conf_frames=cf, conf_merged=cm, frames_total=cf.sum(0), merged_total=cm.sum(0),
                    labelled=labelled, windows=windows, loss_count=count, mean_loss=float(loss.sum() / count) if count else None,
                    min_abs_logit=mabs)

    def launch_count(self) -> int:
        return int(self.L.chd_contact_launch_count(self.h))


class Videos(NamedTuple):
    """A dataset read for the classifier: names, raw keypoints (F_i,25,3), ground truth (T_i,4) or None per video, and
    the preprocessing constants (`ContactNet.preprocess` / `.evaluate`)."""
    names: List[str]
    raw: List[np.ndarray]
    truth: List[Optional[np.ndarray]]
    scale: float
    norm: float


def _subdirs(path: str, prefix: str = "") -> List[str]:
    """contact_data_utils.py / real_video_dataset.py:72: sorted directories, hidden ones skipped."""
    return sorted(d for d in os.listdir(path) if os.path.isdir(os.path.join(path, d)) and d[0] != "." and d.startswith(prefix))


def read_real_videos(data_root: str, dimensions=(1920, 1080)) -> Videos:
    """RealVideoDataset's inputs (real_video_dataset.py:72-120): every video directory of `data_root` with its
    `openpose_result/` and, when present, its `foot_contacts.npy`."""
    vids = _subdirs(data_root)
    raw = load_keypoint_dirs([os.path.join(data_root, v, "openpose_result") for v in vids])
    truth = []
    for v in vids:
        p = os.path.join(data_root, v, "foot_contacts.npy")
        truth.append(np.load(p) if os.path.exists(p) else None)
    return Videos(vids, raw, truth, video_scale(dimensions), TRAIN_NORMALIZATION)


def data_layout(data_root: str) -> str:
    """"real" when a video directory of `data_root` has an `openpose_result/`, "synthetic" when a
    `<character>/<motion>/view*` directory exists; ValueError otherwise."""
    subs = _subdirs(data_root)
    if any(os.path.isdir(os.path.join(data_root, s, "openpose_result")) for s in subs):
        return "real"
    for s in subs:
        for m in _subdirs(os.path.join(data_root, s)):
            if _subdirs(os.path.join(data_root, s, m), "view"):
                return "synthetic"
    raise ValueError("%s holds neither real videos (<video>/openpose_result/) nor the synthetic dataset "
                     "(<character>/<motion>/view<k>/)" % data_root)


SPLITS = ("train", "test", "val")


def synthetic_splits(n_characters: int, n_motions: int, n_views: int, train_frac: float = 0.8) -> Dict[str, List[int]]:
    """OpenPoseDataset's split (openpose_dataset.py:214-238): the motions of each character in turn are shuffled by one
    stream seeded with 0 (np.random.seed(0) + np.random.shuffle, here a RandomState(0)), the first 80 % train, then half
    of the rest test, the remainder val; every view of a motion follows it.  Global sequence indices (character-major,
    then motion, then view) in the reference's order."""
    rs = np.random.RandomState(0)
    out = {k: [] for k in SPLITS}
    for c in range(n_characters):
        inds = np.arange(n_motions)
        rs.shuffle(inds)
        ntr = int(train_frac * n_motions)
        nte = (n_motions - ntr) // 2
        for k, part in zip(SPLITS, (inds[:ntr], inds[ntr:ntr + nte], inds[ntr + nte:])):
            for m in part:
                g = (c * n_motions + int(m)) * n_views
                out[k] += range(g, g + n_views)
    return out


class SyntheticVideos(NamedTuple):
    """`read_synthetic_videos`: the videos of one split plus what the split and the normalisation were made from."""
    videos: Videos
    splits: Dict[str, List[int]]          # global sequence indices of train / test / val
    all_names: List[str]                  # "<character>/<motion>/view<k>" of every sequence, global order
    median: float
    num_frames: int


def read_synthetic_videos(data_root: str, split: str = "test") -> SyntheticVideos:
    """OpenPoseDataset(data_root, split, overlap_test=True) (openpose_dataset.py:126-269) up to the preprocessing: sorted
    character / motion / view directories, the frame count from the `*.png` of the first view, one foot_contacts.npy per
    motion shared by its views, the seeded split, and as `norm` the median MidHip -> LBigToe distance over the raw
    keypoints of every sequence of every split (:212, :368-382).  `scale` is 1: no padding, no 1280 scaling.  Raises
    ValueError for a tree whose characters differ in motion count, whose motions differ in view count, or a sequence whose
    keypoint count differs from the frame count (the reference assumes all three)."""
    if split not in SPLITS:
        raise ValueError("split must be one of %s" % ", ".join(SPLITS))
    chars = _subdirs(data_root)
    if not chars:
        raise ValueError("no character directories under %s" % data_root)
    motions = [[os.path.join(data_root, c, m) for m in _subdirs(os.path.join(data_root, c))] for c in chars]
    if not motions[0] or any(len(m) != len(motions[0]) for m in motions):
        raise ValueError("every character of %s must hold the same number of motions" % data_root)
    mdirs = [m for ms in motions for m in ms]
    views = [_subdirs(m, "view") for m in mdirs]
    if not views[0] or any(len(v) != len(views[0]) for v in views):
        raise ValueError("every motion of %s must hold the same number of view directories" % data_root)
    v0 = os.path.join(mdirs[0], views[0][0])
    num_frames = len([f for f in os.listdir(v0) if f[0] != "." and f.split(".")[-1] == "png"])
    names, kdirs, cpaths = [], [], []
    for m, vs in zip(mdirs, views):
        for v in vs:
            names.append("/".join(os.path.normpath(os.path.join(m, v)).split(os.sep)[-3:]))
            kdirs.append(os.path.join(m, "keypoints_" + v))
            cpaths.append(os.path.join(m, "foot_contacts.npy"))
    raw = load_keypoint_dirs(kdirs)
    for n, r in zip(names, raw):
        if r.shape[0] != num_frames:
            raise ValueError("%s: %d keypoint files but %d frames (*.png in %s)" % (n, r.shape[0], num_frames, v0))
    dists = np.concatenate([np.linalg.norm(r[:, 8, :2] - r[:, 19, :2], axis=1) for r in raw])    # MidHip, LBigToe
    median = float(np.median(dists))
    splits = synthetic_splits(len(chars), len(motions[0]), len(views[0]))
    sel = splits[split]
    truth = {p: np.load(p) for p in set(cpaths[i] for i in sel) if os.path.exists(p)}
    vids = Videos([names[i] for i in sel], [raw[i] for i in sel], [truth.get(cpaths[i]) for i in sel], 1.0, median)
    return SyntheticVideos(vids, splits, names, median, num_frames)


def read_videos(data_root: str, real_data: bool = False, dimensions=(1920, 1080)):
    """What test.py --full-video reads: (layout, Videos).  `real_data` or a root in the real-video layout -> every video
    (`read_real_videos`); otherwise the test split of the synthetic dataset (`read_synthetic_videos`)."""
    layout = "real" if real_data else data_layout(data_root)
    if layout == "real":
        return layout, read_real_videos(data_root, dimensions)
    return layout, read_synthetic_videos(data_root, "test").videos


def detect_contacts(data_root: str, out_root: str, state_dict, dimensions=(1920, 1080), precision: str = "fp32") -> List[str]:
    """`test.py --data D --out O --full-video --save-contacts --real-data`: for every video directory of D with an
    `openpose_result/` writes O/contact_results/<video>/foot_contacts.npy (int64, F x 4), test.py:143-152.
    `precision`: numerical mode of the network (see `ContactNet`)."""
    precision_code(precision)
    vids = read_real_videos(data_root, dimensions)
    net = ContactNet(state_dict, precision=precision)
    labels, _ = net.detect(vids.raw, dimensions)
    return save_contacts(out_root, vids.names, labels)


def save_contacts(out_root: str, names: Sequence[str], labels: Sequence[np.ndarray]) -> List[str]:
    """out_root/contact_results/<name>/foot_contacts.npy (int64, F x 4) per video, test.py:143-152."""
    written = []
    for n, lab in zip(names, labels):
        od = os.path.join(out_root, "contact_results", n)
        os.makedirs(od, exist_ok=True)
        np.save(os.path.join(od, "foot_contacts"), lab.astype(np.int64))
        written.append(os.path.join(od, "foot_contacts.npy"))
    return written
