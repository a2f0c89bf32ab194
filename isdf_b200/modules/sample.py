"""Pixel / ray / depth sampling -- host-side mirror of reference isdf/modules/sample.py.

Random numbers are drawn by torch in the reference's order (sample.py:15-16, 123, 160-162) so a
seeded run reproduces the reference's batch; the gathers, back-projection and depth placement run
in the K1 kernels (isdfb_gather_rays / isdfb_sample_rays)."""
import torch

from ..engine import Engine, make_camera

_ENGINES = {}


def _engine(device):
    """A tiny context for the sampling kernels when the caller has no SDFMap engine at hand."""
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("isdf_b200.sample runs on CUDA tensors only (got %s); there is no CPU path" % device)
    key = (device.type, device.index if device.index is not None else torch.cuda.current_device())
    if key not in _ENGINES:
        _ENGINES[key] = Engine(device, 1, 128, 1, 1.0, 1.0, precision="fp32", max_points=128)
    return _ENGINES[key]


def sample_pixels(n_rays, n_frames, h, w, device):
    """Uniform pixels, n_rays PER FRAME (sample.py:11-21)."""
    total = n_rays * n_frames
    indices_h = torch.randint(0, h, (total,), device=device)
    indices_w = torch.randint(0, w, (total,), device=device)
    indices_b = torch.arange(n_frames, device=device).repeat_interleave(n_rays)
    return indices_b, indices_h, indices_w


def camera_from_dirs(dirs_C):
    """Recover (fx, fy, cx, cy, H, W) from a reference-style dirs_C [1,H,W,3] tensor."""
    _, H, W, _ = dirs_C.shape
    x0, x1 = float(dirs_C[0, 0, 0, 0]), float(dirs_C[0, 0, 1, 0])
    y0, y1 = float(dirs_C[0, 0, 0, 1]), float(dirs_C[0, 1, 0, 1])
    fx, fy = 1.0 / (x1 - x0), 1.0 / (y1 - y0)
    return make_camera(fx, fy, -x0 * fx, -y0 * fy, H, W)


def get_batch_data(depth_batch, T_WC_batch, dirs_C, indices_b, indices_h, indices_w, norm_batch=None,
                   get_masks=False, cam=None, engine=None, frame_map=None, normals_use_frame_map=False):
    """Depth / normal / pose / camera direction of the sampled pixels, invalid rays dropped
    (sample.py:24-74).  `dirs_C` may be the reference's [1,H,W,3] tensor or None when `cam` is given:
    directions are recomputed from (h, w) instead of being read from HBM."""
    eng = engine or _engine(depth_batch.device)
    if cam is None:
        cam = camera_from_dirs(dirs_C)
    depth_s, norm_s, valid = eng.gather_rays(depth_batch, norm_batch, indices_b, indices_h, indices_w, cam,
                                             frame_map=frame_map, normals_use_frame_map=normals_use_frame_map)
    keep = valid.bool()
    depth_s = depth_s[keep]                  # boolean compaction: data-dependent size (host sync, as in the reference)
    if norm_s is not None:
        norm_s = norm_s[keep]
    indices_b, indices_h, indices_w = indices_b[keep], indices_h[keep], indices_w[keep]
    fsel = indices_b if frame_map is None else torch.as_tensor(frame_map, device=indices_b.device)[indices_b]
    T_WC_sample = T_WC_batch[fsel]
    x = (indices_w.float() - cam.cx) / cam.fx
    y = (indices_h.float() - cam.cy) / cam.fy
    dirs_C_sample = torch.stack((x, y, torch.ones_like(x)), dim=-1)
    masks = None
    if get_masks:
        masks = torch.zeros(depth_batch.shape if frame_map is None else (len(frame_map),) + tuple(depth_batch.shape[1:]),
                            device=depth_batch.device)
        masks[indices_b, indices_h, indices_w] = 1
    return (dirs_C_sample, depth_s, norm_s, T_WC_sample, masks, indices_b, indices_h, indices_w)


def stratified_sample(min_depth, max_depth, n_rays, device, n_stratified_samples, bin_length=None):
    """One uniform sample per depth bin (sample.py:77-128).  Small torch helper kept for API parity; the
    training path computes the same values inside isdfb_sample_rays."""
    if n_stratified_samples is not None:
        n_bins = n_stratified_samples
        if torch.is_tensor(max_depth):
            span = (max_depth - min_depth)[:, None]
            edges = torch.linspace(0, 1, n_bins + 1, device=device)[None, :].repeat(n_rays, 1) * span
            edges = edges + (min_depth[:, None] if torch.is_tensor(min_depth) else min_depth)
            bin_length = span / n_bins
        else:
            edges = torch.linspace(min_depth, max_depth, n_bins + 1, device=device)[None, :]
            bin_length = (max_depth - min_depth) / n_bins
    elif bin_length is not None:
        edges = torch.arange(min_depth, max_depth, bin_length, device=device)[None, :]
        n_bins = edges.size(1) - 1
    else:
        raise ValueError("pass n_stratified_samples or bin_length")
    return edges[..., :-1] + torch.rand(n_rays, n_bins, device=device) * bin_length


def sample_along_rays(T_WC, min_depth, max_depth, n_stratified_samples, n_surf_samples, dirs_C,
                      gt_depth=None, grad=False, engine=None, rng_device=None):
    """3-D sample points along back-projected rays (sample.py:131-178): surface sample, clamped
    Gaussian near-surface samples (CPU RNG in the reference -- quirk Q6, kept), stratified samples."""
    if grad:
        raise NotImplementedError("grad=True (pose refinement) is not part of the hot path")
    dev = T_WC.device
    eng = engine or _engine(dev)
    dirs_C = dirs_C.reshape(-1, 3)
    R = dirs_C.shape[0]
    rd = rng_device or dev
    with_surf = gt_depth is not None and n_surf_samples > 0
    n_surf = n_surf_samples if with_surf else 0       # gt_depth=None: stratified samples only (sample.py:158)
    S = n_stratified_samples + n_surf
    if R == 0:
        return torch.empty(0, S, 3, device=dev), torch.empty(0, S, device=dev)

    def per_ray(v):
        return v.to(dev).float().reshape(-1).expand(R) if torch.is_tensor(v) else torch.full((R,), float(v), device=dev)

    far = per_ray(max_depth)
    near = per_ray(min_depth) if torch.is_tensor(min_depth) else None
    if not torch.is_tensor(max_depth) and near is None:
        near = per_ray(min_depth)                     # scalar/scalar: same bins up to the rounding of linspace
    u = torch.rand(R, n_stratified_samples, device=rd).to(dev)
    off = torch.normal(torch.zeros(R, n_surf - 1), 0.1).to(dev) if n_surf > 1 else None      # CPU RNG (quirk Q6)
    lin = torch.linspace(0, 1, n_stratified_samples + 1).to(dev)
    cam = make_camera(1.0, 1.0, 0.0, 0.0, 1, 1)           # unused: directions are given explicitly
    T = T_WC.reshape(-1, 4, 4)
    ib = None if T.shape[0] == R else torch.zeros(R, dtype=torch.int64, device=dev)       # one pose for all rays
    pc, z, _, _ = eng.sample_rays(T, ib, None, None, gt_depth if with_surf else None, u, off, lin,
                                  n_stratified_samples, n_surf, cam, 0.0 if near is not None else float(min_depth),
                                  0.0, dirs_C_in=dirs_C, far=far, near=near)
    return pc, z
