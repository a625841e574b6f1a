"""GPU tests of the contact classifier's 3xTF32 tensor-core mode (`chd_contact_set_precision(net, CHD_CONTACT_TF32X3)`):
accuracy against an fp64 forward and against the fp32 mode, labels, slabs, mode switching, determinism."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

SLAB = 16384          # windows per slab (chd_contact.cu)


def forward_fp64(sd, windows, eps=1e-5):
    """windows (..., 9, 13, 3) fp32 -> logits (..., 5, 4): the eval-mode network of oracle/contact.py:forward_torch
    evaluated in float64."""
    x = np.asarray(windows, dtype=np.float64).reshape(-1, 351)
    lin, bn = [0, 3, 6, 10, 13], [1, 4, 7, 11]
    for i, li in enumerate(lin):
        x = x @ np.asarray(sd["model.%d.weight" % li], np.float64).T + np.asarray(sd["model.%d.bias" % li], np.float64)
        if i < 4:
            p = {k: np.asarray(sd["model.%d.%s" % (bn[i], k)], np.float64) for k in ("weight", "bias", "running_mean", "running_var")}
            x = np.maximum((x - p["running_mean"]) / np.sqrt(p["running_var"] + eps) * p["weight"] + p["bias"], 0.0)
    return x.reshape(np.shape(windows)[:-3] + (5, 4))


def check_labels(labels, ref_labels, ref_logits, seq_lens, max_risky):
    """labels equal ref_labels except in videos with an fp64 logit within 1e-4 of zero (the rule of
    test_contact_gpu.py::test_large_batch_against_torch_reference), and at most `max_risky` such videos."""
    risky = 0
    for i in range(len(seq_lens)):
        L = int(seq_lens[i])
        if not np.array_equal(labels[i, :L], ref_labels[i]):
            assert np.abs(ref_logits[i]).min() < 1e-4, i
            risky += 1
        assert (labels[i, L:] == 0).all()
    assert risky <= max_risky


def test_golden_clips_against_fp64(chd):
    from make_contact_golden import contact_weights
    from oracle import contact as oc
    g = dict(np.load(os.path.join(HERE, "golden", "contact", "contact_golden.npz")))
    names = [str(n) for n in g["names"]]
    frames = np.stack([g["proc_" + n] for n in names])
    lens = g["seq_lens"].astype(np.int32)
    sd = contact_weights(0)
    ref = forward_fp64(sd, oc.windows_from_frames(frames))
    net32 = chd.contact.ContactNet(sd)
    _, lg32, _ = net32.forward(frames, lens, want_logits=True)
    net = chd.contact.ContactNet(sd, precision="tf32x3")
    assert net.precision == "tf32x3"
    labels, logits, mabs = net.forward(frames, lens, want_logits=True)
    e32, etc = float(np.abs(lg32 - ref).max()), float(np.abs(logits - ref).max())
    print("max |logit - fp64|: fp32 %.3g, tf32x3 %.3g" % (e32, etc))
    np.testing.assert_allclose(logits, ref, rtol=0, atol=5e-5)
    check_labels(labels, [g["contacts_" + n] for n in names], ref, lens, max_risky=len(names))
    assert labels.dtype == np.int64 and mabs > 0


def _batch(kind):
    from make_contact_golden import contact_weights, synth_keypoints
    if kind == "48-videos":
        return contact_weights(1), [synth_keypoints(1000 + i, 60 + (i % 7)) for i in range(48)]
    rng = np.random.default_rng(7)        # 200 videos of 90..110 frames: two slabs, the second one ragged
    return contact_weights(2), [synth_keypoints(3000 + i, int(rng.integers(90, 111))) for i in range(200)]


@pytest.mark.parametrize("kind", ["48-videos", "two-slabs"])
def test_large_batches_against_fp32_mode(chd, kind):
    from oracle import contact as oc
    sd, raw = _batch(kind)
    net32 = chd.contact.ContactNet(sd)
    frames, lens = net32.preprocess(raw)
    lab32, lg32, _ = net32.forward(frames, lens, want_logits=True)
    net = chd.contact.ContactNet(sd, precision="tf32x3")
    n0 = net.launch_count()
    labels, logits, _ = net.forward(frames, lens, want_logits=True)
    total = logits.shape[0] * logits.shape[1]
    slabs = (total + SLAB - 1) // SLAB
    if kind == "two-slabs":
        assert slabs == 2 and total % SLAB != 0
    assert net.launch_count() - n0 == 5 * slabs + 1               # per slab: gather, three GEMMs, tail; one vote
    print("%s: %d windows, max |tf32x3 - fp32| %.3g" % (kind, total, float(np.abs(logits - lg32).max())))
    np.testing.assert_allclose(logits, lg32, rtol=0, atol=5e-5)
    ref = forward_fp64(sd, oc.windows_from_frames(frames))
    check_labels(labels, [lab32[i, :lens[i]] for i in range(len(raw))], ref, lens, max_risky=1)
    det, _ = net.detect(raw)                                          # one-call path in the same mode: same labels
    for i in range(len(raw)):
        np.testing.assert_array_equal(det[i], labels[i, :lens[i]])
    labels2, logits2, _ = net.forward(frames, lens, want_logits=True)  # deterministic: bitwise the same
    np.testing.assert_array_equal(logits2, logits)
    np.testing.assert_array_equal(labels2, labels)


def test_mode_switching(chd):
    from make_contact_golden import contact_weights
    g = dict(np.load(os.path.join(HERE, "golden", "contact", "contact_golden.npz")))
    names = [str(n) for n in g["names"]]
    frames = np.stack([g["proc_" + n] for n in names])
    lens = g["seq_lens"].astype(np.int32)
    sd = contact_weights(0)
    lab0, lg0, m0 = chd.contact.ContactNet(sd).forward(frames, lens, want_logits=True)
    net = chd.contact.ContactNet(sd)
    net.set_precision("tf32x3")
    n0 = net.launch_count()
    _, lgt, _ = net.forward(frames, lens, want_logits=True)
    assert net.launch_count() - n0 == 6                              # one slab: six launches, as in fp32 mode
    assert not np.array_equal(lgt, lg0)                               # the fast mode did run
    net.set_precision("fp32")
    lab1, lg1, m1 = net.forward(frames, lens, want_logits=True)
    np.testing.assert_array_equal(lg1, lg0)
    np.testing.assert_array_equal(lab1, lab0)
    assert m1 == m0
    assert net.L.chd_contact_set_precision(net.h, C.c_int32(7)) == -1
    assert net.L.chd_contact_set_precision(None, C.c_int32(1)) == -1
    with pytest.raises(ValueError):
        net.set_precision("tf32")
    with pytest.raises(ValueError):
        chd.contact.ContactNet(sd, precision="bf16")
    assert net.precision == "fp32"


def test_single_nine_frame_video(chd):
    from make_contact_golden import contact_weights, synth_keypoints
    from oracle import contact as oc
    sd = contact_weights(0)
    raw = [synth_keypoints(55, 9)]
    net = chd.contact.ContactNet(sd, precision="tf32x3")
    frames, lens = net.preprocess(raw)
    labels, logits, mabs = net.forward(frames, lens, want_logits=True)
    assert logits.shape == (1, 1, 5, 4)
    np.testing.assert_allclose(logits, forward_fp64(sd, oc.windows_from_frames(frames)), rtol=0, atol=5e-5)
    det, _ = net.detect(raw)
    np.testing.assert_array_equal(det[0], labels[0, :9])
