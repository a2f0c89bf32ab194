"""Per-step time of Trainer.step() at the shape of the realsense_franka_offline config (1280 x 720 frames, E = 465 with
hidden_layers_block 3, 200 rays per window frame, 27 samples per ray), with the card name and power limit of the run.
The sequence is tests/golden/franka_case.py's synthetic one; all of its 8 frames are keyframes, so every step draws the
window (5 of 8).  For each precision: the step time Trainer.step() reports (CUDA events around the step; median and
mean over the timed steps), and the wall time of the same number of back-to-back steps without the per-step
synchronisation.  Also the host-to-keyframe ingest of one frame (read, get_data, add_frame).  Prints one JSON line.
    python tools/franka_time.py [steps]"""
import contextlib
import io
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import eval_time as ET  # noqa: E402
from tests.golden import franka_case as FC  # noqa: E402

WARMUP = 50


def run(seq, precision, rng_mode, steps):
    from isdf.modules import trainer
    np.random.seed(1)
    torch.manual_seed(1)
    with contextlib.redirect_stdout(io.StringIO()):
        tr = trainer.Trainer("cuda:0", FC.config(seq), precision=precision, rng_mode=rng_mode)
        t0 = time.perf_counter()
        for k in range(FC.PARAMS["n_frames"]):
            tr.last_is_keyframe = True
            tr.add_frame(tr.get_data([k]))
        torch.cuda.synchronize()
        ingest_ms = (time.perf_counter() - t0) * 1e3 / FC.PARAMS["n_frames"]
        tr.last_is_keyframe = True
        for _ in range(WARMUP):
            tr.step()
        per = [tr.step()[1] for _ in range(steps)]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            losses, _ = tr.step(sync=False)
        torch.cuda.synchronize()
        wall_ms = (time.perf_counter() - t0) * 1e3 / steps
    return {"step_ms_median": float(np.median(per)), "step_ms_mean": float(np.mean(per)),
            "back_to_back_ms": wall_ms, "ingest_ms_per_frame": ingest_ms, "keyframes": len(tr.frames),
            "total_loss": float(losses["total_loss"])}


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 500
    res = {"card": ET.card(), "shape": "1280x720, E=465, block 3, 5 x 200 rays x 27 samples", "steps": steps}
    with tempfile.TemporaryDirectory() as tmp:
        seq = FC.write_sequence(os.path.join(tmp, "seq"))
        for precision, rng_mode in (("bf16x3g", "fast"), ("fp32", "reference")):
            res["%s_%s" % (precision, rng_mode)] = {k: (round(v, 4) if isinstance(v, float) else v)
                                                    for k, v in run(seq, precision, rng_mode, steps).items()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
