"""Thin torch <-> C-ABI adapter: owns one `isdfb_ctx`, checks tensors, passes raw device pointers
and the caller's current CUDA stream.  PyTorch is used for device memory and streams only."""
import ctypes as C

import torch

from . import _lib


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _f32(t, name, device):
    if t is None:
        return None
    if t.device != device:
        raise ValueError("%s is on %s, engine is on %s" % (name, t.device, device))
    if t.dtype != torch.float32:
        raise TypeError("%s must be float32, got %s" % (name, t.dtype))
    return t.contiguous()


def _i64(t, name, device):
    if t is None:
        return None
    if t.device != device:
        raise ValueError("%s is on %s, engine is on %s" % (name, t.device, device))
    return t.to(torch.int64).contiguous()


class Engine:
    """One CUDA context of the iSDF hot path (model shape + workspaces)."""

    def __init__(self, device, n_freqs, hidden, block, scale_input, scale_output, transform=None,
                 precision="fp32", max_points=32768):
        self.lib = _lib.load()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("isdf_b200 runs on CUDA devices only (got %s); there is no CPU path" % device)
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        cfg = _lib.ModelCfg()
        cfg.n_freqs, cfg.hidden, cfg.block = int(n_freqs), int(hidden), int(block)
        cfg.scale_input, cfg.scale_output = float(scale_input), float(scale_output)
        cfg.has_transform = 0 if transform is None else 1
        if transform is not None:
            tr = torch.as_tensor(transform, dtype=torch.float32).cpu()
            flat = tr[:3, :4].reshape(-1).tolist()
            for i, v in enumerate(flat):
                cfg.transform[i] = v
        if precision not in _lib.PRECISIONS:
            raise ValueError("precision must be one of %s" % list(_lib.PRECISIONS))
        cfg.precision = _lib.PRECISIONS[precision]
        cfg.max_points = int(max_points)
        self.precision = precision
        self.n_freqs, self.hidden, self.block = int(n_freqs), int(hidden), int(block)
        self._ctx = C.c_void_p()
        rc = self.lib.isdfb_create(C.byref(cfg), self.device.index, C.byref(self._ctx))
        if rc != 0:
            msg = self.lib.isdfb_last_error(None)
            raise _lib.IsdfbError("isdfb_create failed (%d): %s" % (rc, msg.decode() if msg else "?"))
        self.n_params = int(self.lib.isdfb_param_count(self._ctx))
        self.embedding_size = int(self.lib.isdfb_embedding_size(self._ctx))

    def __deepcopy__(self, memo):
        return None          # contexts are not copyable; owners re-create them lazily

    def __del__(self):
        try:
            if getattr(self, "_ctx", None) is not None and self._ctx.value:
                self.lib.isdfb_destroy(self._ctx)
                self._ctx = C.c_void_p()
        except Exception:
            pass

    # ------------------------------------------------------------------
    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _ck(self, rc):
        _lib.check(rc, self._ctx)

    @property
    def launches(self):
        return int(self.lib.isdfb_launch_count(self._ctx))

    # ---- weights -----------------------------------------------------
    def pack_weights(self, flat):
        flat = _f32(flat, "params", self.device)
        if flat.numel() != self.n_params:
            raise ValueError("expected %d parameters, got %d" % (self.n_params, flat.numel()))
        self._ck(self.lib.isdfb_pack_weights(self._ctx, _ptr(flat), self._stream()))

    # ---- K1 ----------------------------------------------------------
    def gather_rays(self, depth, normals, ib, ih, iw, cam, frame_map=None, normals_use_frame_map=False):
        dev = self.device
        depth = _f32(depth, "depth", dev)
        normals = _f32(normals, "normals", dev)
        ib, ih, iw = _i64(ib, "indices_b", dev), _i64(ih, "indices_h", dev), _i64(iw, "indices_w", dev)
        frame_map = _i64(frame_map, "frame_map", dev)
        n = ib.numel()
        d_out = torch.empty(n, dtype=torch.float32, device=dev)
        n_out = torch.empty(n, 3, dtype=torch.float32, device=dev) if normals is not None else None
        valid = torch.empty(n, dtype=torch.uint8, device=dev)
        self._ck(self.lib.isdfb_gather_rays(self._ctx, _ptr(depth), _ptr(normals), _ptr(frame_map),
                                            1 if normals_use_frame_map else 0, _ptr(ib), _ptr(ih), _ptr(iw), n,
                                            C.byref(cam), _ptr(d_out), _ptr(n_out), _ptr(valid), self._stream()))
        return d_out, n_out, valid

    def sample_rays(self, T_WC, ib, ih, iw, depth_sample, u_strat, n_near, lin, n_strat, n_surf, cam,
                    min_depth, dist_behind, frame_map=None, dirs_C_in=None, far=None, near=None):
        dev = self.device
        T_WC = _f32(T_WC, "T_WC", dev)
        ib, ih, iw = _i64(ib, "indices_b", dev), _i64(ih, "indices_h", dev), _i64(iw, "indices_w", dev)
        dirs_C_in = _f32(dirs_C_in, "dirs_C", dev)
        far = _f32(far, "max_depth", dev)
        near = _f32(near, "min_depth", dev)
        frame_map = _i64(frame_map, "frame_map", dev)
        depth_sample = _f32(depth_sample, "depth_sample", dev)
        u_strat = _f32(u_strat, "u_strat", dev)
        n_near = _f32(n_near, "n_near", dev)
        lin = _f32(lin, "lin", dev)
        R = depth_sample.numel() if depth_sample is not None else far.numel()
        S = n_strat + n_surf
        if u_strat.shape != (R, n_strat):
            raise ValueError("u_strat must be [%d,%d]" % (R, n_strat))
        if n_surf > 1 and n_near.shape != (R, n_surf - 1):
            raise ValueError("n_near must be [%d,%d]" % (R, n_surf - 1))
        pc = torch.empty(R, S, 3, dtype=torch.float32, device=dev)
        z = torch.empty(R, S, dtype=torch.float32, device=dev)
        dirs_C = torch.empty(R, 3, dtype=torch.float32, device=dev)
        T_s = torch.empty(R, 4, 4, dtype=torch.float32, device=dev)
        self._ck(self.lib.isdfb_sample_rays(self._ctx, _ptr(T_WC), _ptr(frame_map), _ptr(ib), _ptr(ih), _ptr(iw),
                                            _ptr(dirs_C_in), _ptr(depth_sample), _ptr(far), _ptr(near), _ptr(u_strat), _ptr(n_near), _ptr(lin), R,
                                            int(n_strat), int(n_surf), C.byref(cam), float(min_depth),
                                            float(dist_behind), _ptr(pc), _ptr(z), _ptr(dirs_C), _ptr(T_s),
                                            self._stream()))
        return pc, z, dirs_C, T_s

    def sample_fused(self, depth, normals, T_WC, frame_map, n_frames, n_rays, n_strat, n_surf, cam, min_depth,
                     dist_behind, lin, seed, want_noise=True, normals_use_frame_map=False):
        """K1 fused (fast mode): pixels, gather, depths along rays, world points and the output noise in one
        launch with in-kernel Philox numbers.  Returns the sample dict fields."""
        dev = self.device
        depth, T_WC = _f32(depth, "depth", dev), _f32(T_WC, "T_WC", dev)
        normals = _f32(normals, "normals", dev)
        frame_map = _i64(frame_map, "frame_map", dev)
        lin = _f32(lin, "lin", dev)
        R, S = int(n_frames) * int(n_rays), int(n_strat) + int(n_surf)
        i64 = dict(dtype=torch.int64, device=dev)
        f32 = dict(dtype=torch.float32, device=dev)
        ib, ih, iw = torch.empty(R, **i64), torch.empty(R, **i64), torch.empty(R, **i64)
        pc, z = torch.empty(R, S, 3, **f32), torch.empty(R, S, **f32)
        dirs_C, T_s, d_s = torch.empty(R, 3, **f32), torch.empty(R, 4, 4, **f32), torch.empty(R, **f32)
        n_s = torch.empty(R, 3, **f32) if normals is not None else None
        valid = torch.empty(R, dtype=torch.uint8, device=dev)
        noise = torch.empty(R, S, **f32) if want_noise else None
        inv = torch.empty(1, **f32)
        self._ck(self.lib.isdfb_sample_fused(self._ctx, _ptr(depth), _ptr(normals), _ptr(T_WC), _ptr(frame_map),
                                             1 if normals_use_frame_map else 0, int(n_frames), int(n_rays), int(n_strat),
                                             int(n_surf), C.byref(cam), float(min_depth), float(dist_behind), _ptr(lin),
                                             C.c_uint64(int(seed) & (2 ** 64 - 1)), _ptr(ib), _ptr(ih), _ptr(iw), _ptr(pc),
                                             _ptr(z), _ptr(dirs_C), _ptr(T_s), _ptr(d_s), _ptr(n_s), _ptr(valid), _ptr(noise),
                                             _ptr(inv), self._stream()))
        return dict(pc=pc, z_vals=z, indices_b=ib, indices_h=ih, indices_w=iw, dirs_C_sample=dirs_C, depth_sample=d_s,
                    T_WC_sample=T_s, norm_sample=n_s, ray_valid=valid, noise=noise, inv_count_dev=inv)

    def ingest_normals(self, depth, cam, out=None):
        depth = _f32(depth, "depth", self.device)
        if out is None:
            out = torch.empty(*depth.shape, 3, dtype=torch.float32, device=self.device)
        elif (out.shape != (*depth.shape, 3) or out.dtype != torch.float32 or out.device != self.device
              or not out.is_contiguous()):
            raise ValueError("out must be a contiguous float32 [%s, 3] tensor on %s" % (tuple(depth.shape), self.device))
        self._ck(self.lib.isdfb_ingest_normals(self._ctx, _ptr(depth), C.byref(cam), _ptr(out), self._stream()))
        return out

    def pe_encode(self, x):
        x = _f32(x, "x", self.device)
        n = x.numel() // 3
        out = torch.empty(*x.shape[:-1], self.embedding_size, dtype=torch.float32, device=self.device)
        self._ck(self.lib.isdfb_pe_encode(self._ctx, _ptr(x), n, _ptr(out), self._stream()))
        return out

    # ---- K2 / K3 -----------------------------------------------------
    def forward(self, x, noise=None, noise_std=0.0, want_grad=False):
        dev = self.device
        x = _f32(x, "x", dev)
        shape = x.shape[:-1]
        if x.shape[-1] != 3:
            raise ValueError("points must be [...,3]")
        n = x.numel() // 3
        noise = _f32(noise, "noise", dev)
        if noise is not None and noise.numel() != n:
            raise ValueError("noise must have one value per point")
        sdf = torch.empty(shape, dtype=torch.float32, device=dev)
        if want_grad:
            g = torch.empty(*shape, 3, dtype=torch.float32, device=dev)
            self._ck(self.lib.isdfb_mlp_forward_grad(self._ctx, _ptr(x), _ptr(noise), float(noise_std), n,
                                                     _ptr(sdf), _ptr(g), self._stream()))
            return sdf, g
        self._ck(self.lib.isdfb_mlp_forward(self._ctx, _ptr(x), _ptr(noise), float(noise_std), n, _ptr(sdf),
                                            self._stream()))
        return sdf

    def forward_grid(self, lin, scale=None, transform=None):
        """K2 over the dim^3 lattice x = T (lin_i s_x, lin_j s_y, lin_k s_z), points generated in-kernel (get_sdf_grid)."""
        lin = _f32(lin, "lin", self.device)
        dim = lin.numel()
        sdf = torch.empty(dim, dim, dim, dtype=torch.float32, device=self.device)
        sc = tr = None
        if scale is not None:
            sc = (C.c_float * 3)(*[float(v) for v in torch.as_tensor(scale).reshape(-1).tolist()])
        if transform is not None:
            t = torch.as_tensor(transform, dtype=torch.float32).cpu()[:3, :4].reshape(-1).tolist()
            tr = (C.c_float * 12)(*t)
        self._ck(self.lib.isdfb_mlp_forward_grid(self._ctx, _ptr(lin), int(dim), sc, tr, _ptr(sdf), self._stream()))
        return sdf

    # ---- N4: mesh extraction ------------------------------------------
    def mesh_count(self, sdf):
        """Marching-cubes counts of the lattice sdf [dim,dim,dim] (synchronous): (vertices, faces)."""
        sdf = _f32(sdf, "sdf", self.device)
        dim = sdf.shape[0] if sdf.dim() == 3 else -1
        if sdf.shape != (dim, dim, dim):
            raise ValueError("sdf must be a [dim,dim,dim] lattice, got %s" % (tuple(sdf.shape),))
        nv, nf = C.c_int64(), C.c_int64()
        self._ck(self.lib.isdfb_mesh_count(self._ctx, _ptr(sdf), int(dim), C.byref(nv), C.byref(nf), self._stream()))
        return nv.value, nf.value

    def mesh_emit(self, sdf, verts, faces, scale=None, transform=None):
        """Fill verts [V,3] f32 and faces [F,3] int32 with the mesh of the lattice last passed to mesh_count; the
        capacities are the tensors' row counts."""
        sdf = _f32(sdf, "sdf", self.device)
        for t, nm, dt in ((verts, "verts", torch.float32), (faces, "faces", torch.int32)):
            if t.dtype != dt or t.device != self.device or not t.is_contiguous() or t.dim() != 2 or t.shape[1] != 3:
                raise TypeError("%s must be a contiguous %s [N,3] tensor on %s" % (nm, dt, self.device))
        sc = (C.c_float * 3)(*[float(v) for v in torch.as_tensor(scale).reshape(-1).tolist()]) if scale is not None else None
        tr = None
        if transform is not None:
            tr = (C.c_float * 12)(*torch.as_tensor(transform, dtype=torch.float32).cpu()[:3, :4].reshape(-1).tolist())
        self._ck(self.lib.isdfb_mesh_emit(self._ctx, _ptr(sdf), int(sdf.shape[0]), sc, tr, _ptr(verts), verts.shape[0],
                                          _ptr(faces), faces.shape[0], self._stream()))
        return verts, faces

    def mesh(self, sdf, scale=None, transform=None):
        """Marching cubes at level 0 (draw3D.draw_mesh): vertices [V,3] f32 in the world, faces [F,3] int32."""
        nv, nf = self.mesh_count(sdf)
        verts = torch.empty(nv, 3, dtype=torch.float32, device=self.device)
        faces = torch.empty(nf, 3, dtype=torch.int32, device=self.device)
        return self.mesh_emit(sdf, verts, faces, scale=scale, transform=transform)

    def mesh_cloud(self, depth, T_WC, H_vis, W_vis, fx, fy, cx, cy):
        """Keyframe point cloud of mesh_rec: depth [F,H,W] nearest-resized to (H_vis, W_vis), back-projected with the
        reduced intrinsics, moved to the world.  Returns (cloud [F*H_vis*W_vis, 3], box [6] = min xyz, max xyz)."""
        depth, T_WC = _f32(depth, "depth", self.device), _f32(T_WC, "T_WC", self.device)
        F_, H, W = depth.shape
        if T_WC.shape != (F_, 4, 4):
            raise ValueError("T_WC must be [%d,4,4]" % F_)
        cloud = torch.empty(F_ * int(H_vis) * int(W_vis), 3, dtype=torch.float32, device=self.device)
        box = torch.empty(6, dtype=torch.float32, device=self.device)
        self._ck(self.lib.isdfb_mesh_cloud(self._ctx, _ptr(depth), _ptr(T_WC), F_, H, W, int(H_vis), int(W_vis),
                                           float(fx), float(fy), float(cx), float(cy), _ptr(cloud), _ptr(box),
                                           self._stream()))
        return cloud, box

    def mesh_crop(self, cloud, verts, faces, crop_dist):
        """Keep the faces with a vertex closer than crop_dist to the cloud, then the vertices they use (renumbered in
        order).  Returns (vertices [V',3] f32, faces [F',3] int32)."""
        cloud, verts = _f32(cloud, "cloud", self.device), _f32(verts, "verts", self.device)
        if faces.dtype != torch.int32 or faces.device != self.device:
            raise TypeError("faces must be int32 on %s" % self.device)
        faces = faces.contiguous()
        for t, nm in ((cloud, "cloud"), (verts, "verts"), (faces, "faces")):
            if t.dim() != 2 or t.shape[1] != 3:
                raise ValueError("%s must be [N,3], got %s" % (nm, tuple(t.shape)))
        nv, nf = verts.shape[0], faces.shape[0]
        kv, kf = C.c_int64(), C.c_int64()
        self._ck(self.lib.isdfb_mesh_crop_count(self._ctx, _ptr(cloud), cloud.shape[0], float(crop_dist), _ptr(verts), nv,
                                                _ptr(faces), nf, C.byref(kv), C.byref(kf), self._stream()))
        v_out = torch.empty(kv.value, 3, dtype=torch.float32, device=self.device)
        f_out = torch.empty(kf.value, 3, dtype=torch.int32, device=self.device)
        self._ck(self.lib.isdfb_mesh_crop_emit(self._ctx, _ptr(verts), nv, _ptr(faces), nf, _ptr(v_out), kv.value,
                                               _ptr(f_out), kf.value, self._stream()))
        return v_out, f_out

    # ---- evaluation against a ground-truth SDF -------------------------
    def _lattice_args(self, lattice, origin, spacing, pts, flat):
        """Checks the lattice and the points (float32 or float64, [N,3] if flat else [...,3]) of isdfb_gt_sdf_sample and
        isdfb_gt_sdf_grad.  Returns (lattice, pts, args): the C arguments from the lattice to the point count, and the
        tensors they point into, which the caller holds until the call (they may be contiguous copies)."""
        lattice = _f32(lattice, "lattice", self.device)
        if lattice.dim() != 3:
            raise ValueError("lattice must be [nx,ny,nz], got %s" % (tuple(lattice.shape),))
        if (pts.device != self.device or pts.dtype not in (torch.float32, torch.float64) or (flat and pts.dim() != 2)
                or pts.shape[-1] != 3):
            raise TypeError("pts must be a float32 or float64 %s tensor on %s" % ("[N,3]" if flat else "[...,3]",
                                                                                  self.device))
        pts = pts.contiguous()
        f64 = pts.dtype == torch.float64
        args = (_ptr(lattice), *[int(d) for d in lattice.shape], (C.c_double * 3)(*[float(v) for v in origin]),
                (C.c_double * 3)(*[float(v) for v in spacing]), _ptr(None if f64 else pts), _ptr(pts if f64 else None),
                pts.numel() // 3)
        return lattice, pts, args

    def _pred_gt(self, pred, gt):
        """pred as fp32 [N] and gt as fp64 [N], both contiguous, for the statistics entries."""
        pred = _f32(pred, "pred", self.device).reshape(-1)
        if gt.dtype != torch.float64 or gt.device != self.device or gt.numel() != pred.numel():
            raise TypeError("gt must be float64 on %s with one value per prediction" % self.device)
        return pred, gt.reshape(-1).contiguous()

    def gt_sdf_sample(self, lattice, origin, spacing, pts, fill=0.0):
        """Trilinear interpolation of the fp32 lattice [nx,ny,nz] with nodes i * spacing + origin at pts [...,3]
        (float32 or float64), as scipy's RegularGridInterpolator over sdf_util.get_grid_pts.  Returns (values fp64 [...],
        in-bounds uint8 [...]); out-of-bounds points get `fill`, a NaN coordinate gives NaN and byte 1."""
        lattice, pts, args = self._lattice_args(lattice, origin, spacing, pts, flat=False)
        out = torch.empty(pts.shape[:-1], dtype=torch.float64, device=self.device)
        inb = torch.empty(pts.shape[:-1], dtype=torch.uint8, device=self.device)
        self._ck(self.lib.isdfb_gt_sdf_sample(self._ctx, *args, float(fill), _ptr(out), _ptr(inb), self._stream()))
        return out, inb

    def sdf_error_stats(self, pred, gt, in_bounds, valid=None):
        """The 17 fp64 sums of eval_sdf (device tensor): count, sum |pred - gt|, six bin counts, six bin sums, three
        CHOMP-difference sums, over the points in bounds, valid and with gt != 0."""
        pred, gt = self._pred_gt(pred, gt)
        n = pred.numel()
        masks = []
        for t, nm in ((in_bounds, "in_bounds"), (valid, "valid")):
            if t is not None and (t.device != self.device or t.numel() != n):
                raise ValueError("%s must have one byte per prediction on %s" % (nm, self.device))
            masks.append(None if t is None else t.reshape(-1).to(torch.uint8).contiguous())
        out = torch.empty(17, dtype=torch.float64, device=self.device)
        self._ck(self.lib.isdfb_sdf_error_stats(self._ctx, _ptr(pred), _ptr(gt), _ptr(masks[0]), _ptr(masks[1]), n,
                                                _ptr(out), self._stream()))
        return out

    def points_visible(self, pts, T_CW, depth, fx, fy, cx, cy, trunc):
        """uint8 [N]: 1 iff some frame of depth [F,H,W] (camera-from-world T_CW [F,4,4]) sees the point within trunc
        behind its surface (frustum.is_visible_torch, any over the frames)."""
        pts, T_CW, depth = _f32(pts, "pts", self.device), _f32(T_CW, "T_CW", self.device), _f32(depth, "depth", self.device)
        if pts.dim() != 2 or pts.shape[1] != 3:
            raise ValueError("pts must be [N,3], got %s" % (tuple(pts.shape),))
        F_, H, W = depth.shape
        if T_CW.shape != (F_, 4, 4):
            raise ValueError("T_CW must be [%d,4,4]" % F_)
        vis = torch.empty(pts.shape[0], dtype=torch.uint8, device=self.device)
        self._ck(self.lib.isdfb_points_visible(self._ctx, _ptr(pts), pts.shape[0], _ptr(T_CW), _ptr(depth), F_, H, W,
                                               float(fx), float(fy), float(cx), float(cy), float(trunc), _ptr(vis),
                                               self._stream()))
        return vis

    def gt_sdf_grad(self, lattice, origin, spacing, pts, delta):
        """eval_pts.eval_grad(is_gt_sdf=True) on the lattice of gt_sdf_sample at pts [N,3] (float32 or float64): central
        differences of step delta, NaN where a lookup is outside the lattice or exactly 0.  Returns (grad fp64 [N,3],
        valid uint8 [N], 1 iff no component is NaN)."""
        lattice, pts, args = self._lattice_args(lattice, origin, spacing, pts, flat=True)
        grad = torch.empty(pts.shape[0], 3, dtype=torch.float64, device=self.device)
        valid = torch.empty(pts.shape[0], dtype=torch.uint8, device=self.device)
        self._ck(self.lib.isdfb_gt_sdf_grad(self._ctx, *args, float(delta), _ptr(grad), _ptr(valid), self._stream()))
        return grad, valid

    def sdf_split_stats(self, pred, gt, n_vox):
        """eval_pts.sub_eval's sums (device fp64 [2,17]): row 0 over all points, row 1 over the first n_vox, each in
        sdf_error_stats's layout, with no point left out."""
        pred, gt = self._pred_gt(pred, gt)
        n = pred.numel()
        if not 0 <= int(n_vox) <= n:
            raise ValueError("n_vox %d outside [0, %d]" % (n_vox, n))
        out = torch.empty(2, 17, dtype=torch.float64, device=self.device)
        self._ck(self.lib.isdfb_sdf_split_stats(self._ctx, _ptr(pred), _ptr(gt), n, int(n_vox), _ptr(out),
                                                self._stream()))
        return out

    def grad_cosdist(self, pred, gt, gt_index=None, eps=1e-6):
        """Sum over k of 1 - CosineSimilarity(dim=1, eps)(pred[k], gt[gt_index[k]]) (gt[k] without an index), in fp64
        (device tensor [1]).  pred fp32 [M,3], gt fp64 [N,3], gt_index int64 [M]."""
        pred = _f32(pred, "pred", self.device)
        if pred.dim() != 2 or pred.shape[1] != 3:
            raise ValueError("pred must be [M,3], got %s" % (tuple(pred.shape),))
        if gt.dtype != torch.float64 or gt.device != self.device or gt.dim() != 2 or gt.shape[1] != 3:
            raise TypeError("gt must be a float64 [N,3] tensor on %s" % self.device)
        gt = gt.contiguous()
        m = pred.shape[0]
        if gt_index is not None:
            gt_index = _i64(gt_index, "gt_index", self.device).reshape(-1)
            if gt_index.numel() != m:
                raise ValueError("gt_index must have one entry per prediction")
        elif gt.shape[0] != m:
            raise ValueError("gt must have one row per prediction without gt_index")
        out = torch.empty(1, dtype=torch.float64, device=self.device)
        self._ck(self.lib.isdfb_grad_cosdist(self._ctx, _ptr(pred), _ptr(gt), _ptr(gt_index), m, float(eps), _ptr(out),
                                             self._stream()))
        return out

    # ---- N2 ----------------------------------------------------------
    def bounds_pc(self, pc, z_vals, depth_sample, ray_valid=None):
        """loss.bounds_pc (loss.py:56-89): bounds [R,S] and target directions [R,S,3] (row 0 unused)."""
        dev = self.device
        pc, z_vals = _f32(pc, "pc", dev), _f32(z_vals, "z_vals", dev)
        depth_sample = _f32(depth_sample, "depth_sample", dev)
        R, S = z_vals.shape
        if ray_valid is not None:
            ray_valid = ray_valid.to(torch.uint8).contiguous()
        bounds = torch.empty(R, S, dtype=torch.float32, device=dev)
        vec = torch.empty(R, S, 3, dtype=torch.float32, device=dev)
        self._ck(self.lib.isdfb_bounds_pc(self._ctx, _ptr(pc), _ptr(z_vals), _ptr(depth_sample), _ptr(ray_valid),
                                          R, S, _ptr(bounds), _ptr(vec), self._stream()))
        return bounds, vec

    # ---- K4 ----------------------------------------------------------
    def train_fwd_bwd(self, pc, z_vals, depth_sample, dirs_C, T_WC_sample, norm_sample, noise, loss_cfg,
                      ray_valid=None, want_grad=True, loss_sums=None):
        dev = self.device
        pc = _f32(pc, "pc", dev)
        R, S = pc.shape[0], pc.shape[1]
        z_vals = _f32(z_vals, "z_vals", dev)
        depth_sample = _f32(depth_sample, "depth_sample", dev)
        dirs_C = _f32(dirs_C, "dirs_C_sample", dev)
        T_WC_sample = _f32(T_WC_sample, "T_WC_sample", dev)
        norm_sample = _f32(norm_sample, "norm_sample", dev)
        noise = _f32(noise, "noise", dev)
        if ray_valid is not None:
            ray_valid = ray_valid.to(torch.uint8).contiguous()
        sdf = torch.empty(R, S, dtype=torch.float32, device=dev)
        g = torch.empty(R, S, 3, dtype=torch.float32, device=dev) if want_grad else None
        loss_mat = torch.empty(R, S, dtype=torch.float32, device=dev)
        if loss_sums is None:
            loss_sums = torch.zeros(4, dtype=torch.float32, device=dev)
        self._ck(self.lib.isdfb_train_fwd_bwd(self._ctx, _ptr(pc), _ptr(z_vals), _ptr(depth_sample), _ptr(dirs_C),
                                              _ptr(T_WC_sample), _ptr(norm_sample), _ptr(noise), _ptr(ray_valid),
                                              R, S, C.byref(loss_cfg), _ptr(sdf), _ptr(g), _ptr(loss_mat),
                                              _ptr(loss_sums), self._stream()))
        return sdf, g, loss_mat, loss_sums

    def zero_grad(self):
        self._ck(self.lib.isdfb_zero_grad(self._ctx, self._stream()))

    # ---- C1 fused (gradient exchange over NVLink multicast) ------------------
    def set_grad_exchange(self, local0, local1, mcast0, mcast1, n_floats):
        """Install two symmetric-memory gradient buffers (raw addresses) and their multicast aliases."""
        self._ck(self.lib.isdfb_set_grad_exchange(self._ctx, C.c_void_p(local0), C.c_void_p(local1), C.c_void_p(mcast0),
                                                  C.c_void_p(mcast1), int(n_floats)))

    def select_grad_buffer(self, which):
        self._ck(self.lib.isdfb_select_grad_buffer(self._ctx, int(which)))

    def zero_grad_buffer(self, which):
        self._ck(self.lib.isdfb_zero_grad_buffer(self._ctx, int(which), self._stream()))

    def export_grads(self, out=None):
        if out is None:
            out = torch.empty(self.n_params, dtype=torch.float32, device=self.device)
        self._ck(self.lib.isdfb_export_grads(self._ctx, _ptr(out), self._stream()))
        return out

    def grad_buffer(self):
        """The ctx-internal fp32 gradient buffer as a torch view (for the NCCL all-reduce)."""
        p, n = C.c_void_p(), C.c_int64()
        self._ck(self.lib.isdfb_grad_buffer(self._ctx, C.byref(p), C.byref(n)))
        return _DevView(p.value, n.value, self.device).tensor

    # ---- K5 ----------------------------------------------------------
    def frame_bins(self, loss_mat, ib, ih, iw, n_frames, H, W, factor=8, ray_valid=None):
        dev = self.device
        loss_mat = _f32(loss_mat, "loss_mat", dev)
        ib, ih, iw = _i64(ib, "indices_b", dev), _i64(ih, "indices_h", dev), _i64(iw, "indices_w", dev)
        R, S = loss_mat.shape
        approx = torch.empty(n_frames, factor, factor, dtype=torch.float32, device=dev)
        favg = torch.empty(n_frames, dtype=torch.float32, device=dev)
        if ray_valid is not None:
            ray_valid = ray_valid.to(torch.uint8).contiguous()
        self._ck(self.lib.isdfb_frame_bins(self._ctx, _ptr(loss_mat), _ptr(ray_valid), _ptr(ib), _ptr(ih), _ptr(iw),
                                           R, S, int(n_frames), int(H), int(W), int(factor), _ptr(approx),
                                           _ptr(favg), self._stream()))
        return approx, favg

    def step_finish(self, loss_mat, ib, ih, iw, n_frames, H, W, factor, ray_valid, frame_map, frame_avg_losses,
                    loss_sums, inv_count, means_out):
        """K5 + write-back of the per-keyframe losses + the four loss means (clears loss_sums); see the header."""
        dev = self.device
        R, S = loss_mat.shape
        approx = torch.empty(n_frames, factor, factor, dtype=torch.float32, device=dev)
        favg = torch.empty(n_frames, dtype=torch.float32, device=dev)
        for t, nm in ((frame_avg_losses, "frame_avg_losses"), (loss_sums, "loss_sums"), (inv_count, "inv_count"),
                      (means_out, "means_out")):
            if t is not None and (t.dtype != torch.float32 or t.device != dev or not t.is_contiguous()):
                raise TypeError("%s must be a contiguous float32 tensor on %s" % (nm, dev))
        if ray_valid is not None:
            ray_valid = ray_valid.to(torch.uint8).contiguous()
        self._ck(self.lib.isdfb_step_finish(self._ctx, _ptr(loss_mat), _ptr(ray_valid), _ptr(ib), _ptr(ih), _ptr(iw), R, S,
                                            int(n_frames), int(H), int(W), int(factor), _ptr(approx), _ptr(favg),
                                            _ptr(frame_map), _ptr(frame_avg_losses), _ptr(loss_sums), _ptr(inv_count),
                                            _ptr(means_out), self._stream()))
        return approx, favg

    def select_window(self, frame_avg_losses, n_frames, window_size, seed, out=None):
        """A0 on the device: Gumbel top-k window (see isdfb_select_window)."""
        w = _f32(frame_avg_losses, "frame_avg_losses", self.device)
        if out is None:
            out = torch.empty(window_size, dtype=torch.int64, device=self.device)
        self._ck(self.lib.isdfb_select_window(self._ctx, _ptr(w), int(n_frames), int(window_size),
                                              C.c_uint64(int(seed) & (2 ** 64 - 1)), _ptr(out), self._stream()))
        return out

    # ---- K6 ----------------------------------------------------------
    def adamw(self, params, m, v, step, lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01, grad_scale=1.0):
        for t, nm in ((params, "params"), (m, "exp_avg"), (v, "exp_avg_sq")):
            if t.dtype != torch.float32 or not t.is_contiguous() or t.device != self.device or t.numel() != self.n_params:
                raise ValueError("%s must be a contiguous float32 [%d] tensor on %s" % (nm, self.n_params, self.device))
        self._ck(self.lib.isdfb_adamw(self._ctx, _ptr(params), _ptr(m), _ptr(v), int(step), float(lr), float(beta1),
                                      float(beta2), float(eps), float(weight_decay), float(grad_scale),
                                      self._stream()))


    def adamw_graph(self, params, m, v, lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01, grad_scale=1.0):
        """K6 with the step counter on the device (CUDA-graph capturable)."""
        self._ck(self.lib.isdfb_adamw_graph(self._ctx, _ptr(params), _ptr(m), _ptr(v), float(lr), float(beta1),
                                            float(beta2), float(eps), float(weight_decay), float(grad_scale),
                                            self._stream()))

    def adamw_set_step(self, step):
        self._ck(self.lib.isdfb_adamw_set_step(self._ctx, int(step), self._stream()))

    # ---- kernel timing -------------------------------------------------
    def profile(self, enable):
        self._ck(self.lib.isdfb_profile_enable(self._ctx, 1 if enable else 0))

    def profile_read(self):
        c, d = C.c_double(), C.c_double()
        nc, nd = C.c_int64(), C.c_int64()
        self._ck(self.lib.isdfb_profile_read(self._ctx, C.byref(c), C.byref(d), C.byref(nc), C.byref(nd)))
        return dict(chain_ms=c.value, dw_ms=d.value, n_chain=nc.value, n_dw=nd.value)


class _DevView:
    """Wrap a raw device pointer as a torch tensor through __cuda_array_interface__."""

    def __init__(self, ptr, n, device):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (ptr, False), "version": 2}
        self.tensor = torch.as_tensor(self, device=device)


def make_loss_cfg(trunc_weight, trunc_distance, eik_weight, eik_apply_dist, grad_weight, orien_loss, loss_type,
                  noise_std, inv_count, inv_count_dev=None, bounds=None, grad_vec=None):
    lc = _lib.LossCfg()
    lc.trunc_weight, lc.trunc_distance = float(trunc_weight), float(trunc_distance)
    lc.eik_weight, lc.eik_apply_dist = float(eik_weight), float(eik_apply_dist)
    lc.grad_weight = float(grad_weight)
    lc.orien_loss = 1 if orien_loss else 0
    if loss_type not in ("L1", "L2"):
        raise ValueError("Must be L1 or L2")
    lc.loss_type = 1 if loss_type == "L1" else 2
    lc.noise_std = float(noise_std or 0.0)
    lc.inv_count = float(inv_count)
    lc.inv_count_dev = None
    if inv_count_dev is not None:
        if inv_count_dev.dtype != torch.float32 or not inv_count_dev.is_cuda:
            raise TypeError("inv_count_dev must be a float32 CUDA scalar")
        lc.inv_count_dev = inv_count_dev.data_ptr()
        lc._keepalive = inv_count_dev
    lc.bounds_dev = lc.grad_vec_dev = None
    if (bounds is None) != (grad_vec is None):
        raise ValueError("bounds and grad_vec (the outputs of Engine.bounds_pc) go together")
    if bounds is not None:
        for t, nm in ((bounds, "bounds"), (grad_vec, "grad_vec")):
            if t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous():
                raise TypeError("%s must be a contiguous float32 CUDA tensor" % nm)
        lc.bounds_dev, lc.grad_vec_dev = bounds.data_ptr(), grad_vec.data_ptr()
        lc._keepalive_pc = (bounds, grad_vec)
    return lc


def make_camera(fx, fy, cx, cy, H, W):
    cam = _lib.Camera()
    cam.fx, cam.fy, cam.cx, cam.cy, cam.H, cam.W = float(fx), float(fy), float(cx), float(cy), int(H), int(W)
    return cam


def debug_state(engine):
    """Test helper: decode the tensor-core path's per-tile side arrays into [points, 256] tensors.
    Returns (aux(arr), dwl(arr) (hi + lo), sig(layer)), each -> fp32 [tiles*128, 256]."""
    aux, dhi, dlo, sg = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
    a_st, d_st, tiles = C.c_int64(), C.c_int64(), C.c_int64()
    n_aux, n_dwl = C.c_int32(), C.c_int32()
    engine._ck(engine.lib.isdfb_debug_buffers(engine._ctx, C.byref(aux), C.byref(a_st), C.byref(dhi), C.byref(dlo),
                                              C.byref(d_st), C.byref(n_aux), C.byref(n_dwl), C.byref(tiles), C.byref(sg)))
    T = tiles.value
    aux_t = _DevView(aux.value, a_st.value * n_aux.value, engine.device).tensor.view(n_aux.value, T, 64, 128, 4)

    def raw16(ptr):
        v = _DevView(ptr, d_st.value * n_dwl.value // 4, engine.device).tensor      # fp32 view of the bytes
        return v.view(torch.int16).view(n_dwl.value, T, 8, 32, 16, 8)

    hi = raw16(dhi.value)
    lo = raw16(dlo.value) if dlo.value else None

    def get_aux(arr, n_tiles):
        return aux_t[arr, :n_tiles].permute(0, 2, 1, 3).reshape(n_tiles * 128, 256).clone()

    def get_dwl(arr, n_tiles, part="sum"):
        def dec(x):
            return x[arr, :n_tiles].permute(0, 1, 3, 2, 4).reshape(n_tiles * 128, 256).contiguous().view(torch.bfloat16).float()
        h = dec(hi)
        if part == "hi" or lo is None:
            return h
        return h + dec(lo)

    def get_sig(layer, n_tiles, n_layers):
        v = _DevView(sg.value, d_st.value * n_layers // 4, engine.device).tensor.view(torch.int16)
        v = v.view(n_layers, T, 32, 128, 8)[layer, :n_tiles].permute(0, 2, 1, 3).reshape(n_tiles * 128, 256)
        return (v.to(torch.int32) & 0xFFFF).float() / 65535.0

    return get_aux, get_dwl, get_sig
