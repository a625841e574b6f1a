"""Labelled evaluation of the contact classifier on the host: the synthetic-dataset reader and the numpy scoring checker
against what the reference's own OpenPoseDataset / val_full_video produced (tests/golden/make_contact_eval_golden.py),
and the CLI's choice of layout."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
GOLDEN = os.path.join(HERE, "golden", "contact", "contact_eval_golden.npz")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


@pytest.fixture(scope="module")
def tree(chd, golden, tmp_path_factory):
    c, m, v, f, seed = (int(x) for x in golden["synth_tree"])
    root = str(tmp_path_factory.mktemp("synth"))
    chd.synth.write_contact_dataset(root, c, m, v, f, seed)
    return root


def test_reader_reproduces_split_and_median(chd, golden, tree):
    s = chd.contact.read_synthetic_videos(tree)
    for k in ("train", "test", "val"):
        assert [s.all_names[i] for i in s.splits[k]] == [str(n) for n in golden["synth_" + k]], k
    assert s.median == float(golden["synth_median"])                  # exact: same files, same np.median
    assert s.videos.names == [str(n) for n in golden["synth_test"]] and s.videos.scale == 1.0 and s.videos.norm == s.median
    assert s.num_frames == golden["synth_frames"].shape[1]
    assert all(t is not None and t.shape == (s.num_frames, 4) for t in s.videos.truth)


def test_reader_keypoints_give_golden_frames(chd, golden, tree):
    """The regenerated tree is the one the golden saw: the reference's preprocessing restated (interpolation, / median)
    on the reader's raw keypoints gives the reference's frames bit for bit."""
    from oracle import contact as oc
    s = chd.contact.read_synthetic_videos(tree)
    for i, r in enumerate(s.videos.raw):
        a = oc.interpolate_low_confidence(np.array(r), 0.2)
        a[:, :, :2] /= s.median
        np.testing.assert_array_equal(a, golden["synth_frames"][i])


def test_reader_rejects_frame_count_mismatch(chd, tmp_path):
    root = str(tmp_path)
    chd.synth.write_contact_dataset(root, 1, 2, 1, 12, 3)
    kdir = os.path.join(root, "character00", "motion01", "keypoints_view0")
    os.remove(os.path.join(kdir, sorted(os.listdir(kdir))[-1]))
    with pytest.raises(ValueError, match="character00/motion01/view0: 11 keypoint files but 12 frames"):
        chd.contact.read_synthetic_videos(root)


def truth_of(chd, golden, kind, tree):
    if kind == "synth":
        return chd.contact.read_synthetic_videos(tree).videos.truth
    return [golden.get("real_truth_" + str(n)) for n in golden["real_names"]]


@pytest.mark.parametrize("kind", ["synth", "real"])
def test_oracle_scoring_matches_reference(chd, golden, tree, kind):
    """From the reference's logits: the counts exactly, the loss of every video to 1e-6 relative."""
    from oracle.contact_eval import score
    logits = golden[kind + "_logits"]
    truth = truth_of(chd, golden, kind, tree)
    for v in range(logits.shape[0]):
        loss, cf, cm = score(logits[v], truth[v])
        np.testing.assert_array_equal(cf, golden[kind + "_conf_frames"][v])
        np.testing.assert_array_equal(cm, golden[kind + "_conf_merged"][v])
        assert loss == pytest.approx(golden[kind + "_loss"][v], rel=1e-6, abs=1e-12)
    n = golden[kind + "_count"].sum()
    assert golden[kind + "_loss"].sum() / n == pytest.approx(float(golden[kind + "_mean_loss"]), rel=1e-6)


def test_layout_detection(chd, tree, tmp_path):
    assert chd.contact.data_layout(tree) == "synthetic"
    real = tmp_path / "real"
    (real / "clip" / "openpose_result").mkdir(parents=True)
    assert chd.contact.data_layout(str(real)) == "real"
    (tmp_path / "empty" / "x").mkdir(parents=True)
    with pytest.raises(ValueError, match="neither real videos"):
        chd.contact.data_layout(str(tmp_path / "empty"))
    layout, vids = chd.contact.read_videos(tree)
    assert layout == "synthetic" and len(vids.names) == 4


def test_cli_arguments():
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "scripts"))
    import detect_contacts as dc
    a = dc.parse_args(["--data", "d", "--out", "o", "--weights", "w.npz", "--full-video", "--classify-thresh", "0.7", "--precision", "tf32x3"])
    assert (a.data, a.out, a.weights, a.classify_thresh, a.precision, a.real_data, a.save_contacts) == ("d", "o", "w.npz", 0.7, "tf32x3", False, False)
    with pytest.raises(SystemExit):
        dc.parse_args(["--data", "d", "--out", "o", "--weights", "w", "--precision", "bf16"])
    m = dc.metrics_entry([3, 1, 2, 4])
    assert m["counts"] == {"tp": 3, "fp": 1, "fn": 2, "tn": 4} and m["accuracy"] == 0.7 and m["precision"] == 0.75 and m["recall"] == 0.6
    assert m["confusion_matrix"] == [[0.3, 0.1], [0.2, 0.4]]
