"""GPU test of the drop-in Trainer: the same driver calls as the reference (train.py:102-136) on the
same on-disk sequence, seeded identically, must reproduce the losses the UNMODIFIED reference
Trainer returned on CPU (tests/golden/trainer.pt, made by tests/golden/make_trainer_golden.py)."""
import json
import os

import pytest
import torch

from tests.golden import common as C
from tests.golden import trainer_case as TC

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
MODES = [m for m in os.environ.get("ISDFB_TEST_MODES", "fp32,bf16x3,bf16x3g,bf16").split(",") if m]
# per-step loss tolerance (relative), probe-sdf tolerance (max-abs / max-abs-ref) after 14 AdamW steps
TOL = {"fp32": (2e-4, 2e-3), "bf16x3": (2e-3, 1e-2), "bf16x3g": (2e-3, 1e-2), "bf16": (1e-1, 5e-1)}


@pytest.fixture(scope="module")
def seq(tmp_path_factory):
    root = tmp_path_factory.mktemp("isdf_seq")
    s = TC.write_sequence(str(root))
    cfg_path = os.path.join(str(root), "cfg.json")
    json.dump(TC.config(s), open(cfg_path, "w"))
    return cfg_path


@pytest.mark.parametrize("mode", MODES)
def test_trainer_reproduces_reference_losses(seq, mode, capsys):
    from isdf.modules import trainer            # the alias the reference drivers import (train.py:16)
    gold = torch.load(os.path.join(GOLD, "trainer.pt"), weights_only=False)
    probe = (torch.rand(256, 3, generator=C.gen(70)) - 0.5) * torch.tensor([4.0, 3.0, 6.0])
    out = TC.run_schedule(trainer.Trainer, "cuda:0", seq, probe, precision=mode, rng_mode="reference",
                          rng_device="cpu")
    tol_l, tol_p = TOL[mode]
    assert len(out["losses"]) == len(gold["losses"])
    for i, (a, b) in enumerate(zip(out["losses"], gold["losses"])):
        assert list(a.keys()) == list(b.keys())
        for k in b:
            # rounding noise compounds through the optimiser: allow the tolerance to grow with the step index
            assert abs(a[k] - b[k]) <= tol_l * (1 + i) * max(abs(b[k]), 1e-2), (i, k, a[k], b[k])
    ref = gold["probe_sdf"]
    assert float((out["probe_sdf"] - ref).abs().max() / ref.abs().max()) < tol_p
    assert torch.allclose(out["frame_avg_losses"], gold["frame_avg_losses"], rtol=20 * tol_l, atol=1e-3)


def test_fast_mode_trains_and_never_compacts(seq):
    from isdf.modules import trainer
    import numpy as np
    np.random.seed(1)
    torch.manual_seed(1)
    tr = trainer.Trainer("cuda:0", seq, precision=MODES[0], rng_mode="fast")
    first = last = None
    for k in range(7):
        tr.last_is_keyframe = True
        tr.add_data(tr.get_data([k]))
        for _ in range(6):
            losses, ms = tr.step()
            v = float(losses["total_loss"])
            first = v if first is None else first
            last = v
    assert torch.isfinite(torch.tensor(last)) and last < first
    assert tr.active_pixels["indices_b"].numel() == 5 * 40          # fixed shape: invalid rays are masked
    assert '{:.6f}'.format(losses["total_loss"])                    # train.py:138 formatting works on the lazy value


def test_state_dict_roundtrip_and_optimizer_state(seq):
    from isdf.modules import trainer
    tr = trainer.Trainer("cuda:0", seq, precision=MODES[0])
    tr.last_is_keyframe = True
    tr.add_data(tr.get_data([0]))
    tr.step()
    sd = tr.sdf_map.state_dict()
    assert list(sd.keys())[:2] == ["in_layer.0.weight", "in_layer.0.bias"] and sd["cat_layer.0.weight"].shape == (256, 511)
    osd = tr.optimiser.state_dict()
    assert len(osd["state"]) == 14 and osd["state"][0]["exp_avg"].shape == (256, 255)
    x = torch.rand(50, 3, device="cuda:0")
    a = tr.sdf_map(x)
    tr2 = trainer.Trainer("cuda:0", seq, precision=MODES[0])
    tr2.sdf_map.load_state_dict(sd)
    assert torch.allclose(tr2.sdf_map(x), a, atol=1e-6)
    import copy
    frozen = copy.deepcopy(tr.sdf_map)            # add_frame() does this (trainer.py:576)
    assert torch.allclose(frozen(x), a, atol=1e-6)


def test_fast_mode_keyframe_decision_ignores_invalid_rays(seq):
    """is_keyframe: rays on zero-depth pixels count neither in the numerator nor in the denominator (the reference
    drops them before the mean, sample.py:49-55); the fixed-shape fast mode must reach the same proportion."""
    from isdf.modules import trainer
    import copy
    import io
    import contextlib
    torch.manual_seed(3)
    tr = trainer.Trainer("cuda:0", seq, precision=MODES[0], rng_mode="fast")
    tr.last_is_keyframe = True
    tr.add_data(tr.get_data([0]))
    for _ in range(80):
        tr.step()
    tr.frozen_sdf_map = copy.deepcopy(tr.sdf_map)
    depth = tr.frames.depth_batch[-1].unsqueeze(0).clone()
    T = tr.frames.T_WC_batch[-1].unsqueeze(0)
    tr.n_rays_is_kf = 4000
    props = []
    for frac in (0.0, 0.6):
        d = depth.clone()
        if frac:
            d[:, :, : int(d.shape[2] * frac)] = 0.0            # 60 % of the image without depth
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            tr.is_keyframe(T, d)
        props.append(float(buf.getvalue().split("threshold")[1].split()[0]))
    # the valid part of the image is statistically the same in both runs; without the mask the second proportion
    # would drop by ~60 % of the first
    assert props[0] > 0.2, props                                  # the test discriminates only if the map fits at all
    assert abs(props[0] - props[1]) < 0.08 + 0.15 * props[0], props


def test_graph_replays_keep_the_adamw_step_count(seq, tmp_path):
    """Every replay of the captured fast-mode step advances AdamW's bias-correction step: the checkpoint must say so."""
    from isdf.modules import trainer
    torch.manual_seed(4)
    tr = trainer.Trainer("cuda:0", seq, precision=MODES[0], rng_mode="fast")
    tr.last_is_keyframe = True
    tr.add_data(tr.get_data([0]))
    n = 25
    for _ in range(n):
        tr.step()
    assert tr._graph, "the fast-mode step was not captured"
    osd = tr.optimiser.state_dict()
    assert int(osd["state"][0]["step"]) == n
    # a restored optimiser state re-aligns the device-side counter, graph or not
    tr.optimiser.load_state_dict(osd)
    for _ in range(3):
        tr.step()
    assert int(tr.optimiser.state_dict()["state"][0]["step"]) == n + 3
    # reference optimiser with the same state reproduces one more step (bias corrections depend on `step`)
    ref_params = [p.detach().clone().requires_grad_(True) for p in tr.sdf_map.parameters()]
    opt = torch.optim.AdamW(ref_params, lr=tr.learning_rate, weight_decay=tr.weight_decay)
    opt.load_state_dict(tr.optimiser.state_dict())
    tr.use_graph = False
    tr._step_front()
    g = tr.sdf_map.engine().export_grads()
    off = 0
    for p in ref_params:
        p.grad = g[off:off + p.numel()].view_as(p).clone()
        off += p.numel()
    opt.step()
    tr.optimiser.step()
    for a, b in zip(ref_params, tr.sdf_map.parameters()):
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-7)


def test_configs_with_gt_sdf_dir_take_the_scene_box_from_the_config(seq):
    """replicaCAD.json / scannet.json set dataset.gt_sdf_dir: the reference feeds the oriented scene box of the GT mesh into
    the positional encoding (trainer.py:78-81, 121-129, 421-426).  Here the box comes from b200.scene_box (trimesh is not a
    dependency); without it the constructor must refuse rather than train a different model."""
    from isdf.modules import trainer
    cfg = json.load(open(seq))
    cfg["dataset"]["gt_sdf_dir"] = "/nonexistent/gt_sdfs/apt_2/"
    with pytest.raises(NotImplementedError, match="b200.scene_box"):
        trainer.Trainer("cuda:0", cfg, precision=MODES[0])
    T = C.rigid_transform(21)
    cfg["b200"] = {"scene_box": {"T_extent_to_scene": T.tolist(), "bounds_extents": [6.0, 3.0, 5.0]}}
    tr = trainer.Trainer("cuda:0", cfg, precision=MODES[0], grid_dim=16)
    assert tr.gt_scene and torch.allclose(tr.inv_bounds_transform.cpu(), T)
    assert tr.sdf_map.positional_encoding.transform is tr.inv_bounds_transform      # the PE input transform
    tr.last_is_keyframe = True
    tr.add_data(tr.get_data([0]))
    losses, _ = tr.step()
    assert torch.isfinite(torch.tensor(float(losses["total_loss"])))
    x = torch.rand(64, 3, device="cuda:0")
    a = tr.sdf_map(x)
    tr2 = trainer.Trainer("cuda:0", {k: v for k, v in cfg.items() if k != "b200"} | {"dataset": {k: v for k, v in cfg["dataset"].items()
                                                                                             if k != "gt_sdf_dir"}},
                          precision=MODES[0])
    tr2.sdf_map.load_state_dict(tr.sdf_map.state_dict())
    assert not torch.allclose(tr2.sdf_map(x), a, atol=1e-4)       # same weights, no box -> a different function of x
    assert tr.get_sdf_grid().shape == (16, 16, 16)
