"""Host side of the foot-contact classifier path (reference: scripts/run_detect_contacts.py ->
src/contact_learning/test.py --full-video --save-contacts --real-data).

Keypoint loading (JSON) happens on the host; the dataset preprocessing (padding, scaling, low-confidence
interpolation, normalisation: real_video_dataset.py:132-163, openpose_dataset.py:49-121), window construction, the MLP
and the vote aggregation run in hand-written CUDA behind `chd_contact_*` (include/chd.h).  No CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, List, Sequence

import numpy as np

from .phys import load_lib

TRAIN_DIM = (1280, 720)                      # real_video_dataset.py:17
TRAIN_NORMALIZATION = 200.4160302695367      # real_video_dataset.py:18
WINDOW, PRED = 9, 5
LIN_IDS, BN_IDS = [0, 3, 6, 10, 13], [1, 4, 7, 11]
DIMS = [351, 1024, 512, 128, 32, 20]


def load_keypoint_files(files: Sequence[str], num_joints: int = 25, threads: int = 0) -> np.ndarray:
    """Many OpenPose `*_keypoints.json` files -> (len(files), J, 3) fp64 through the native threaded reader
    (`chd_openpose_load`, csrc/chd_openpose.cpp); bit-identical to openpose_utils.py:48-66 applied per file."""
    L = load_lib()
    out = np.empty((len(files), num_joints, 3), dtype=np.float64)
    arr = (C.c_char_p * len(files))(*[os.fsencode(f) for f in files])
    L.chd_openpose_load.argtypes = [C.POINTER(C.c_char_p), C.c_int32, C.c_int32, C.c_void_p, C.c_int32]
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
        self.L = load_lib()
        L = self.L
        L.chd_contact_create.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_int32, C.POINTER(C.c_void_p)]
        L.chd_contact_destroy.argtypes = [C.c_void_p]
        L.chd_contact_destroy.restype = None
        L.chd_contact_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.chd_contact_preprocess.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
        L.chd_contact_detect.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
        L.chd_contact_launch_count.argtypes = [C.c_void_p]
        L.chd_contact_launch_count.restype = C.c_int64
        L.chd_contact_set_precision.argtypes = [C.c_void_p, C.c_int32]
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

    def preprocess(self, raw: Sequence[np.ndarray], dimensions=(1920, 1080)):
        """RealVideoDataset.__init__ on the device (`chd_contact_preprocess`): list of raw (F_i,25,3) keypoints ->
        (frames (V,Fmax,25,3) fp64, seq_lens (V,) int32), bit identical to the reference's numpy result."""
        cat, offs = concat_videos(raw)
        V, Fmax = len(raw), int(np.diff(offs).max())
        frames = np.zeros((V, Fmax, 25, 3))
        lens = np.zeros(V, dtype=np.int32)
        rc = self.L.chd_contact_preprocess(self.h, cat.ctypes.data, offs.ctypes.data, V, int(dimensions[0]), frames.ctypes.data, lens.ctypes.data)
        if rc != 0:
            raise RuntimeError("chd_contact_preprocess failed with code %d" % rc)
        return frames, lens

    def detect(self, raw: Sequence[np.ndarray], dimensions=(1920, 1080), cat=None, offs=None):
        """raw keypoints -> list of (F_i,4) int64 foot-contact labels (`chd_contact_detect`: preprocessing, windows,
        network, votes on the device; one upload, one download).  `cat` / `offs` may carry a pre-concatenated (e.g.
        page-locked) buffer."""
        if cat is None:
            cat, offs = concat_videos(raw)
        V = len(offs) - 1
        lab = np.zeros((int(offs[-1]), 4), dtype=np.int64)
        mabs = np.zeros(1, dtype=np.float32)
        rc = self.L.chd_contact_detect(self.h, cat.ctypes.data, offs.ctypes.data, V, int(dimensions[0]), lab.ctypes.data, mabs.ctypes.data)
        if rc != 0:
            raise RuntimeError("chd_contact_detect failed with code %d" % rc)
        return [lab[offs[i]:offs[i + 1]] for i in range(V)], float(mabs[0])

    def launch_count(self) -> int:
        return int(self.L.chd_contact_launch_count(self.h))


def detect_contacts(data_root: str, out_root: str, state_dict, dimensions=(1920, 1080), precision: str = "fp32") -> List[str]:
    """`test.py --data D --out O --full-video --save-contacts --real-data`: for every video directory of D with an
    `openpose_result/` writes O/contact_results/<video>/foot_contacts.npy (int64, F x 4), test.py:143-152.
    `precision`: numerical mode of the network (see `ContactNet`)."""
    precision_code(precision)
    vids = sorted(d for d in os.listdir(data_root) if os.path.isdir(os.path.join(data_root, d)) and d[0] != ".")
    raw = load_keypoint_dirs([os.path.join(data_root, v, "openpose_result") for v in vids])
    net = ContactNet(state_dict, precision=precision)
    labels, _ = net.detect(raw, dimensions)
    written = []
    for i, v in enumerate(vids):
        od = os.path.join(out_root, "contact_results", v)
        os.makedirs(od, exist_ok=True)
        np.save(os.path.join(od, "foot_contacts"), labels[i].astype(np.int64))
        written.append(os.path.join(od, "foot_contacts.npy"))
    return written
