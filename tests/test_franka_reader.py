"""CPU tests of the realsense_franka_offline reader (isdf_b200.datasets.dataset.RealsenseFrankaOffline): what it returns
for the synthetic Franka sequence of tests/golden/franka_case.py against what the UNMODIFIED reference reader returned
for the same files (tests/golden/franka.pt, made by tests/golden/make_golden_franka.py), and its refusals."""
import hashlib
import os

import numpy as np
import pytest
import torch

from tests.golden import franka_case as FC

GOLD = os.path.join(os.path.dirname(__file__), "golden", "franka.pt")


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, weights_only=False)


@pytest.fixture(scope="module")
def seq(tmp_path_factory, gold):
    return FC.write_sequence(str(tmp_path_factory.mktemp("franka_seq")), gold["params"])


def reader(seq_dir, params, traj="traj.txt"):
    from isdf_b200.datasets import dataset as ds
    return ds.RealsenseFrankaOffline(seq_dir, traj_file=None if traj is None else os.path.join(seq_dir, traj),
                                     rgb_transform=ds.bgr_to_rgb,
                                     depth_transform=ds.depth_scale_filter(1.0 / params["depth_scale"],
                                                                           params["max_depth"]),
                                     col_ext=".jpg")


def test_generator_rebuilds_the_fixture_files(gold, seq):
    assert gold["params"] == FC.PARAMS
    for k, f in enumerate(gold["frames"]):
        assert sha(np.load(os.path.join(seq, "depth", "%05d.npy" % k))) == f["raw_depth_sha"], k


def test_reader_matches_the_reference_reader(gold, seq):
    """Depth and T bitwise; the image equal after the same cv2 JPEG decode (BGR -> RGB)."""
    p = gold["params"]
    rd = reader(seq, p)
    assert len(rd) == gold["len"] == p["n_frames"]
    for k, f in enumerate(gold["frames"]):
        s = rd[k]
        assert set(s) == {"image", "depth", "T"}
        assert s["T"].dtype == np.float64 and np.array_equal(s["T"], f["T"].numpy()), k
        d, im = s["depth"], s["image"]
        assert (str(d.dtype), d.shape) == (f["depth_dtype"], f["depth_shape"]) == ("float32", (p["H"], p["W"]))
        assert (str(im.dtype), im.shape) == (f["image_dtype"], f["image_shape"]) == ("uint8", (p["H"], p["W"], 3))
        for (r, c), dc, ic in zip(FC.CROPS, f["depth_crops"], f["image_crops"]):
            assert np.array_equal(d[r, c], dc.numpy()), k
            assert np.array_equal(im[r, c], ic.numpy()), k
        assert sha(d) == f["depth_sha"], k
        assert sha(im) == f["image_sha"], k
        # the fixture covers both ends of the depth filter: missing depth and depth beyond max_depth read as 0
        raw = np.load(os.path.join(seq, "depth", "%05d.npy" % k))
        assert (raw == 0).any() and (raw > 1000 * p["max_depth"]).any()
        assert np.array_equal(d == 0, (raw == 0) | (raw > 1000 * p["max_depth"]))


def test_numpy_index_and_relative_root(gold, seq, monkeypatch):
    """Indices as numpy integers (Trainer.get_data passes them) and a root relative to the current directory."""
    rd = reader(seq, gold["params"])
    a = rd[np.int64(3)]
    monkeypatch.chdir(os.path.dirname(seq))
    rel = reader(os.path.basename(seq), gold["params"])
    b = rel[3]
    assert np.array_equal(a["depth"], b["depth"]) and np.array_equal(a["image"], b["image"])
    assert os.getcwd() == os.path.dirname(seq)                    # the reader leaves the working directory alone


def test_missing_frames_and_poses_are_refused(gold, seq, tmp_path):
    import shutil
    p = gold["params"]
    with pytest.raises(ValueError, match="traj_file"):
        reader(seq, p, traj=None)
    with pytest.raises(FileNotFoundError):
        reader(seq, p, traj="no_such_traj.txt")
    rd = reader(seq, p)
    with pytest.raises(FileNotFoundError):
        rd[p["n_frames"]]                                          # a pose row is not enough: the frame files are missing
    cut = tmp_path / "cut"
    shutil.copytree(seq, cut)
    os.remove(cut / "rgb" / "00002.jpg")
    os.remove(cut / "depth" / "00004.npy")
    rd = reader(str(cut), p)
    assert rd[1]["depth"].shape == (p["H"], p["W"])
    with pytest.raises(FileNotFoundError, match="00002"):
        rd[2]
    with pytest.raises(FileNotFoundError, match="00004"):
        rd[4]


@pytest.mark.reference
def test_reference_reader_returns_the_same_arrays(gold, seq):
    """With the reference present: its reader run live over the same files, whole arrays compared."""
    from oracle import ref_shim
    if not ref_shim.available():
        pytest.skip("the reference is not present")
    ref = ref_shim.load()
    dataset, tf = ref["trainer"].dataset, ref["trainer"].image_transforms
    compose = ref["trainer"].transforms.Compose
    p = gold["params"]
    cwd = os.getcwd()
    try:
        rr = dataset.RealsenseFrankaOffline(
            seq, traj_file=os.path.join(seq, "traj.txt"), rgb_transform=compose([tf.BGRtoRGB()]),
            depth_transform=compose([tf.DepthScale(1.0 / p["depth_scale"]), tf.DepthFilter(p["max_depth"])]),
            col_ext=".jpg")
    finally:
        os.chdir(cwd)                                              # the reference constructor changes directory
    rd = reader(seq, p)
    assert len(rr) == len(rd)
    for k in (0, 5):
        a, b = rd[k], rr[k]
        for key in ("image", "depth", "T"):
            assert a[key].dtype == b[key].dtype and np.array_equal(a[key], b[key]), (k, key)
