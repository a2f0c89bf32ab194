"""Golden fixture for the realsense_franka_offline reader: writes the synthetic sequence of franka_case.py and reads it
back with the UNMODIFIED reference RealsenseFrankaOffline (isdf/datasets/dataset.py:123-173) and the reference's own
transforms, BGRtoRGB and DepthScale + DepthFilter, composed as its Trainer.load_data does (trainer.py:458-463, 496-501).
    python tests/golden/make_golden_franka.py      Writes tests/golden/franka.pt:
  params     franka_case.PARAMS (the tests rebuild the same files from it)
  frames     per frame: T (fp64 [4,4]); SHA-256 of the depth (fp32 [H,W], metres, far values zeroed) and of the RGB
             image (uint8 [H,W,3]) as the reference returned them, and both arrays in full on franka_case.CROPS; the
             SHA-256 of the uint16 depth written to disk (to catch a change of the generator itself)
  len        len() of the reader
A full 1280 x 720 frame is 3.7 MB of depth and 2.8 MB of image, so the whole arrays are kept as digests only.
The reference constructor changes the working directory (os.chdir to the script's directory); it is restored here."""
import hashlib
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from tests.golden import franka_case as FC  # noqa: E402


def sha(a):
    a = np.ascontiguousarray(a)
    return hashlib.sha256(a.tobytes()).hexdigest()


def describe_frame(sample, raw_depth):
    depth, image, T = sample["depth"], sample["image"], sample["T"]
    return {"T": torch.from_numpy(np.array(T, dtype=np.float64)),
            "depth_sha": sha(depth), "depth_dtype": str(depth.dtype), "depth_shape": tuple(depth.shape),
            "image_sha": sha(image), "image_dtype": str(image.dtype), "image_shape": tuple(image.shape),
            "depth_crops": [torch.from_numpy(np.array(depth[r, c])) for r, c in FC.CROPS],
            "image_crops": [torch.from_numpy(np.array(image[r, c])) for r, c in FC.CROPS],
            "raw_depth_sha": sha(raw_depth)}


def main():
    ref = ref_shim.load()
    dataset, tf = ref["trainer"].dataset, ref["trainer"].image_transforms
    compose = ref["trainer"].transforms.Compose
    p = FC.PARAMS
    seq = FC.write_sequence(tempfile.mkdtemp(prefix="isdf_franka_golden_"))
    cwd = os.getcwd()
    try:
        rd = dataset.RealsenseFrankaOffline(
            seq, traj_file=os.path.join(seq, "traj.txt"), rgb_transform=compose([tf.BGRtoRGB()]),
            depth_transform=compose([tf.DepthScale(1.0 / p["depth_scale"]), tf.DepthFilter(p["max_depth"])]),
            col_ext=".jpg")
    finally:
        os.chdir(cwd)
    frames = [describe_frame(rd[k], np.load(os.path.join(seq, "depth", "%05d.npy" % k))) for k in range(len(rd))]
    out = {"params": dict(p), "frames": frames, "len": len(rd)}
    torch.save(out, os.path.join(HERE, "franka.pt"))
    for k, f in enumerate(frames):
        d = rd[k]["depth"]
        print(k, "valid %.3f" % float((d > 0).mean()), "range [%.3f, %.3f]" % (d[d > 0].min(), d.max()), f["depth_sha"][:12])
    print("wrote franka.pt")


if __name__ == "__main__":
    main()
