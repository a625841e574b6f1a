"""Labelled evaluation of the contact classifier on the GPU (`chd_contact_detect` with truth, `chd_k_contact_score`)
against the counts and loss the reference's own val_full_video produced (tests/golden/make_contact_eval_golden.py)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(os.path.join(HERE, "golden", "contact", "contact_eval_golden.npz")))


@pytest.fixture(scope="module")
def tree(chd, golden, tmp_path_factory):
    c, m, v, f, seed = (int(x) for x in golden["synth_tree"])
    root = str(tmp_path_factory.mktemp("synth"))
    chd.synth.write_contact_dataset(root, c, m, v, f, seed)
    return root


@pytest.fixture(scope="module")
def weights():
    from make_contact_golden import contact_weights
    return contact_weights(0)


def datasets(chd, golden, tree):
    s = chd.contact.read_synthetic_videos(tree).videos
    names = [str(n) for n in golden["real_names"]]
    real = chd.contact.Videos(names, [golden["real_raw_" + n] for n in names], [golden.get("real_truth_" + n) for n in names],
                              chd.contact.video_scale(), chd.contact.TRAIN_NORMALIZATION)
    return {"synth": s, "real": real}


def check_against_golden(res, golden, kind):
    np.testing.assert_array_equal(res["conf_frames"], golden[kind + "_conf_frames"])
    np.testing.assert_array_equal(res["conf_merged"], golden[kind + "_conf_merged"])
    np.testing.assert_allclose(res["loss_sum"], golden[kind + "_loss"], rtol=1e-5, atol=0)
    assert res["loss_count"] == golden[kind + "_count"].sum()
    assert res["mean_loss"] == pytest.approx(float(golden[kind + "_mean_loss"]), rel=1e-5)


def test_synthetic_preprocessing_bit_exact(chd, golden, tree, weights):
    v = chd.contact.read_synthetic_videos(tree).videos
    net = chd.contact.ContactNet(weights)
    frames, lens = net.preprocess(v.raw, scale=v.scale, norm=v.norm)
    np.testing.assert_array_equal(frames, golden["synth_frames"])
    assert (lens == golden["synth_frames"].shape[1]).all()


@pytest.mark.parametrize("kind", ["synth", "real"])
@pytest.mark.parametrize("precision", ["fp32", "tf32x3"])
def test_counts_and_loss_match_reference(chd, golden, tree, weights, kind, precision):
    """Per-frame and merged counts equal the reference's, loss to 1e-5 relative; the real set pads a shorter video and
    carries truth longer than, shorter than and missing for its keypoints.  tf32x3 gives the same counts here."""
    v = datasets(chd, golden, tree)[kind]
    net = chd.contact.ContactNet(weights, precision=precision)
    res = net.evaluate(v.raw, v.truth, v.scale, v.norm)
    check_against_golden(res, golden, kind)
    det, _ = net.detect(v.raw) if kind == "real" else (None, None)
    if det is not None:                       # evaluate's labels are detect's
        for a, b in zip(res["labels"], det):
            np.testing.assert_array_equal(a, b)


def test_labels_equal_detect_and_forward(chd, golden, tree, weights):
    v = datasets(chd, golden, tree)["synth"]
    net = chd.contact.ContactNet(weights)
    res = net.evaluate(v.raw, v.truth, v.scale, v.norm)
    frames, lens = net.preprocess(v.raw, scale=v.scale, norm=v.norm)
    lab, logits, _ = net.forward(frames, lens, want_logits=True)
    for i in range(len(v.raw)):
        np.testing.assert_array_equal(res["labels"][i], lab[i, :lens[i]])
    np.testing.assert_allclose(logits, golden["synth_logits"], rtol=0, atol=2e-5)


def test_per_video_results_independent_of_batch(chd, golden, tree, weights):
    v = datasets(chd, golden, tree)["synth"]
    net = chd.contact.ContactNet(weights)
    full = net.evaluate(v.raw, v.truth, v.scale, v.norm, classify_thresh=0.3)
    for i in range(len(v.raw)):
        one = net.evaluate([v.raw[i]], [v.truth[i]], v.scale, v.norm, classify_thresh=0.3)
        assert one["loss_sum"][0].tobytes() == full["loss_sum"][i].tobytes()
        np.testing.assert_array_equal(one["conf_frames"][0], full["conf_frames"][i])
        np.testing.assert_array_equal(one["conf_merged"][0], full["conf_merged"][i])
        np.testing.assert_array_equal(one["labels"][0], full["labels"][i])


def test_classify_thresh_and_oracle(chd, golden, tree, weights):
    """Per-frame counts follow classify_thresh, merged counts keep the 0.5 vote; both equal the numpy checker's on the
    device logits."""
    from oracle.contact_eval import score
    v = datasets(chd, golden, tree)["real"]
    net = chd.contact.ContactNet(weights)
    res = net.evaluate(v.raw, v.truth, v.scale, v.norm, classify_thresh=0.7)
    frames, lens = net.preprocess(v.raw)
    _, logits, _ = net.forward(frames, lens, want_logits=True)
    for i in range(len(v.raw)):
        loss, cf, cm = score(logits[i], v.truth[i], thresh=0.7)
        np.testing.assert_array_equal(res["conf_frames"][i], cf)
        np.testing.assert_array_equal(res["conf_merged"][i], cm)
        np.testing.assert_allclose(res["loss_sum"][i], loss, rtol=1e-6)
    np.testing.assert_array_equal(res["conf_merged"], golden["real_conf_merged"])
    assert res["conf_frames"][:, :, 0].sum() < golden["real_conf_frames"][:, :, 0].sum()     # fewer predicted contacts


def test_launch_counts(chd, golden, tree, weights):
    v = datasets(chd, golden, tree)["synth"]
    net = chd.contact.ContactNet(weights)
    frames, lens = net.preprocess(v.raw, scale=v.scale, norm=v.norm)
    l0 = net.launch_count()
    net.forward(frames, lens)
    assert net.launch_count() - l0 == 6            # gather, three tiled layers, tail, vote: unchanged
    l0 = net.launch_count()
    net.evaluate(v.raw, v.truth, v.scale, v.norm)
    assert net.launch_count() - l0 == 9            # prep, the forward's six, score, pack


def test_cli_end_to_end(chd, tree, weights, tmp_path):
    w = str(tmp_path / "w.npz")
    np.savez(w, **weights)
    out = str(tmp_path / "out")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "detect_contacts.py"), "--data", tree, "--out", out, "--weights", w,
                        "--full-video", "--save-contacts"], capture_output=True, text=True, check=True)
    for s in ("TEST RESULTS", "Mean Loss:", "----- Pred Frame 4 ------", "F1 Score:", "FULL VIDEO MERGED RESULTS"):
        assert s in r.stdout
    m = json.load(open(os.path.join(out, "test_metrics.json")))
    v = chd.contact.read_synthetic_videos(tree).videos
    res = chd.contact.ContactNet(weights).evaluate(v.raw, v.truth, v.scale, v.norm)
    assert m["mean_loss"] == res["mean_loss"] and m["labelled_videos"] == 4
    assert [m["pred_frames"][p]["counts"]["tp"] for p in range(5)] == res["frames_total"][:, 0].tolist()
    assert m["merged"]["counts"]["fn"] == int(res["merged_total"][2])
    for i, n in enumerate(v.names):
        np.testing.assert_array_equal(np.load(os.path.join(out, "contact_results", n, "foot_contacts.npy")), res["labels"][i])
