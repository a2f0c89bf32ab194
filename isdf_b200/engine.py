"""Thin torch <-> C-ABI adapter: owns one `isdfb_ctx`, checks every tensor it hands to C (`Engine._arg`), passes raw
device pointers and the caller's current CUDA stream.  PyTorch is used for device memory and streams only."""
import ctypes as C

import torch

from . import _lib

F32, F64, I32, I64, U8 = torch.float32, torch.float64, torch.int32, torch.int64, torch.uint8
_SMALL_INTS = (torch.uint8, torch.int8, torch.int16, torch.int32)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _shape_ok(t, shape, rows):
    if isinstance(shape, int):
        ok = t.numel() == shape
    elif shape is None:
        ok = True
    else:
        want = shape[1:] if shape[0] is ... else shape
        got = t.shape[max(t.dim() - len(want), 0):] if shape[0] is ... else t.shape
        ok = len(got) == len(want) and all(w is None or w == g for w, g in zip(want, got))
    return ok and (rows == 0 or (t.dim() > 0 and t.shape[0] >= rows))


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

    def _arg(self, t, name, dtype, shape=None, rows=0, as_is=False):
        """`t` as a C entry may receive it, from its metadata alone (no device value is read); None stays None.
        dtype: one dtype or a tuple of them.  shape: an element count, or a tuple of sizes in which None matches any
        size and a leading ... any leading axes.  rows: the least size of axis 0, for a buffer reached through an index
        or a count.  as_is: the entry gets `t` itself, as an output or in-place state must (a copy would lose the
        write); otherwise `t` is made contiguous, an integer index becomes int64 and a bool mask uint8.  Raises
        TypeError for the dtype, ValueError for the device, shape or layout."""
        if t is None:
            return None
        if t.device != self.device:
            raise ValueError("%s is on %s, engine is on %s" % (name, t.device, self.device))
        dtypes = dtype if isinstance(dtype, tuple) else (dtype,)
        convert = not as_is and ((dtype == I64 and t.dtype in _SMALL_INTS) or (dtype == U8 and t.dtype == torch.bool))
        if t.dtype not in dtypes and not convert:
            raise TypeError("%s must be %s, got %s" % (name, " or ".join(map(str, dtypes)), t.dtype))
        if not _shape_ok(t, shape, rows):
            want = "%d elements" % shape if isinstance(shape, int) else "[%s]" % ", ".join(
                "..." if s is ... else "*" if s is None else str(s) for s in shape)
            raise ValueError("%s must be %s%s, got %s" % (name, want, " with >= %d rows" % rows if rows else "",
                                                          list(t.shape)))
        if as_is and not t.is_contiguous():
            raise ValueError("%s must be contiguous: the entry writes into it" % name)
        return t if as_is else t.to(dtypes[0] if convert else t.dtype).contiguous()

    @property
    def launches(self):
        return int(self.lib.isdfb_launch_count(self._ctx))

    # ---- weights -----------------------------------------------------
    def pack_weights(self, flat):
        flat = self._arg(flat, "params", F32, self.n_params)
        self._ck(self.lib.isdfb_pack_weights(self._ctx, _ptr(flat), self._stream()))

    # ---- K1 ----------------------------------------------------------
    def gather_rays(self, depth, normals, ib, ih, iw, cam, frame_map=None, normals_use_frame_map=False):
        dev = self.device
        ib = self._arg(ib, "indices_b", I64, (None,))
        n = ib.shape[0]
        ih, iw = self._arg(ih, "indices_h", I64, (n,)), self._arg(iw, "indices_w", I64, (n,))
        depth = self._arg(depth, "depth", F32, (None, cam.H, cam.W))
        normals = self._arg(normals, "normals", F32, (None, cam.H, cam.W, 3))
        frame_map = self._arg(frame_map, "frame_map", I64, (None,))
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
        R = depth_sample.numel() if depth_sample is not None else far.numel()
        S = n_strat + n_surf
        depth_sample, far = self._arg(depth_sample, "depth_sample", F32, R), self._arg(far, "max_depth", F32, R)
        near = self._arg(near, "min_depth", F32, R)
        ib, ih = self._arg(ib, "indices_b", I64, R), self._arg(ih, "indices_h", I64, R)
        iw = self._arg(iw, "indices_w", I64, R)
        T_WC = self._arg(T_WC, "T_WC", F32, (R if ib is None else None, 4, 4))
        dirs_C_in = self._arg(dirs_C_in, "dirs_C", F32, (R, 3))
        frame_map = self._arg(frame_map, "frame_map", I64, (None,))
        u_strat = self._arg(u_strat, "u_strat", F32, (R, n_strat))
        n_near = self._arg(n_near, "n_near", F32, (R, max(n_surf - 1, 0)))
        lin = self._arg(lin, "lin", F32, (None,), rows=n_strat + 1)
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
        frame_map = self._arg(frame_map, "frame_map", I64, (None,), rows=n_frames)
        F_ = n_frames if frame_map is None else 0          # keyframe rows the slots address without a frame_map
        depth = self._arg(depth, "depth", F32, (None, cam.H, cam.W), rows=F_)
        T_WC = self._arg(T_WC, "T_WC", F32, (None, 4, 4), rows=F_)
        normals = self._arg(normals, "normals", F32, (None, cam.H, cam.W, 3),
                            rows=F_ if normals_use_frame_map else n_frames)
        lin = self._arg(lin, "lin", F32, (None,), rows=n_strat + 1)
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
        depth = self._arg(depth, "depth", F32, (cam.H, cam.W))
        if out is None:
            out = torch.empty(cam.H, cam.W, 3, dtype=torch.float32, device=self.device)
        out = self._arg(out, "out", F32, (cam.H, cam.W, 3), as_is=True)
        self._ck(self.lib.isdfb_ingest_normals(self._ctx, _ptr(depth), C.byref(cam), _ptr(out), self._stream()))
        return out

    def pe_encode(self, x):
        x = self._arg(x, "x", F32, (..., 3))
        n = x.numel() // 3
        out = torch.empty(*x.shape[:-1], self.embedding_size, dtype=torch.float32, device=self.device)
        self._ck(self.lib.isdfb_pe_encode(self._ctx, _ptr(x), n, _ptr(out), self._stream()))
        return out

    # ---- K2 / K3 -----------------------------------------------------
    def forward(self, x, noise=None, noise_std=0.0, want_grad=False):
        dev = self.device
        x = self._arg(x, "x", F32, (..., 3))
        shape = x.shape[:-1]
        n = x.numel() // 3
        noise = self._arg(noise, "noise", F32, n)
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
        lin = self._arg(lin, "lin", F32, (None,))
        dim = lin.shape[0]
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
    def _cube(self, sdf):
        d = sdf.shape[0] if sdf.dim() else 0
        return self._arg(sdf, "sdf", F32, (d, d, d))

    def mesh_count(self, sdf):
        """Marching-cubes counts of the lattice sdf [dim,dim,dim] (synchronous): (vertices, faces)."""
        sdf = self._cube(sdf)
        nv, nf = C.c_int64(), C.c_int64()
        self._ck(self.lib.isdfb_mesh_count(self._ctx, _ptr(sdf), sdf.shape[0], C.byref(nv), C.byref(nf),
                                           self._stream()))
        return nv.value, nf.value

    def mesh_emit(self, sdf, verts, faces, scale=None, transform=None):
        """Fill verts [V,3] f32 and faces [F,3] int32 with the mesh of the lattice last passed to mesh_count; the
        capacities are the tensors' row counts."""
        sdf = self._cube(sdf)
        verts = self._arg(verts, "verts", F32, (None, 3), as_is=True)
        faces = self._arg(faces, "faces", I32, (None, 3), as_is=True)
        sc = (C.c_float * 3)(*[float(v) for v in torch.as_tensor(scale).reshape(-1).tolist()]) if scale is not None else None
        tr = None
        if transform is not None:
            tr = (C.c_float * 12)(*torch.as_tensor(transform, dtype=torch.float32).cpu()[:3, :4].reshape(-1).tolist())
        self._ck(self.lib.isdfb_mesh_emit(self._ctx, _ptr(sdf), sdf.shape[0], sc, tr, _ptr(verts), verts.shape[0],
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
        depth = self._arg(depth, "depth", F32, (None, None, None))
        F_, H, W = depth.shape
        T_WC = self._arg(T_WC, "T_WC", F32, (F_, 4, 4))
        cloud = torch.empty(F_ * int(H_vis) * int(W_vis), 3, dtype=torch.float32, device=self.device)
        box = torch.empty(6, dtype=torch.float32, device=self.device)
        self._ck(self.lib.isdfb_mesh_cloud(self._ctx, _ptr(depth), _ptr(T_WC), F_, H, W, int(H_vis), int(W_vis),
                                           float(fx), float(fy), float(cx), float(cy), _ptr(cloud), _ptr(box),
                                           self._stream()))
        return cloud, box

    def mesh_crop(self, cloud, verts, faces, crop_dist):
        """Keep the faces with a vertex closer than crop_dist to the cloud, then the vertices they use (renumbered in
        order).  Returns (vertices [V',3] f32, faces [F',3] int32)."""
        cloud = self._arg(cloud, "cloud", F32, (None, 3))
        verts, faces = self._arg(verts, "verts", F32, (None, 3)), self._arg(faces, "faces", I32, (None, 3))
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
    @staticmethod
    def _lattice_args(lattice, origin, spacing, pts):
        """The C arguments of isdfb_gt_sdf_sample and isdfb_gt_sdf_grad from the lattice to the point count."""
        f64 = pts.dtype == F64
        return (_ptr(lattice), *lattice.shape, (C.c_double * 3)(*[float(v) for v in origin]),
                (C.c_double * 3)(*[float(v) for v in spacing]), _ptr(None if f64 else pts), _ptr(pts if f64 else None),
                pts.numel() // 3)

    def gt_sdf_sample(self, lattice, origin, spacing, pts, fill=0.0):
        """Trilinear interpolation of the fp32 lattice [nx,ny,nz] with nodes i * spacing + origin at pts [...,3]
        (float32 or float64), as scipy's RegularGridInterpolator over sdf_util.get_grid_pts.  Returns (values fp64 [...],
        in-bounds uint8 [...]); out-of-bounds points get `fill`, a NaN coordinate gives NaN and byte 1."""
        lattice = self._arg(lattice, "lattice", F32, (None, None, None))
        pts = self._arg(pts, "pts", (F32, F64), (..., 3))
        out = torch.empty(pts.shape[:-1], dtype=torch.float64, device=self.device)
        inb = torch.empty(pts.shape[:-1], dtype=torch.uint8, device=self.device)
        self._ck(self.lib.isdfb_gt_sdf_sample(self._ctx, *self._lattice_args(lattice, origin, spacing, pts),
                                              float(fill), _ptr(out), _ptr(inb), self._stream()))
        return out, inb

    def sdf_error_stats(self, pred, gt, in_bounds, valid=None):
        """The 17 fp64 sums of eval_sdf (device tensor): count, sum |pred - gt|, six bin counts, six bin sums, three
        CHOMP-difference sums, over the points in bounds, valid and with gt != 0."""
        n = pred.numel()
        pred, gt = self._arg(pred, "pred", F32, n), self._arg(gt, "gt", F64, n)
        in_bounds, valid = self._arg(in_bounds, "in_bounds", U8, n), self._arg(valid, "valid", U8, n)
        out = torch.empty(17, dtype=torch.float64, device=self.device)
        self._ck(self.lib.isdfb_sdf_error_stats(self._ctx, _ptr(pred), _ptr(gt), _ptr(in_bounds), _ptr(valid), n,
                                                _ptr(out), self._stream()))
        return out

    def points_visible(self, pts, T_CW, depth, fx, fy, cx, cy, trunc):
        """uint8 [N]: 1 iff some frame of depth [F,H,W] (camera-from-world T_CW [F,4,4]) sees the point within trunc
        behind its surface (frustum.is_visible_torch, any over the frames)."""
        pts = self._arg(pts, "pts", F32, (None, 3))
        depth = self._arg(depth, "depth", F32, (None, None, None))
        F_, H, W = depth.shape
        T_CW = self._arg(T_CW, "T_CW", F32, (F_, 4, 4))
        vis = torch.empty(pts.shape[0], dtype=torch.uint8, device=self.device)
        self._ck(self.lib.isdfb_points_visible(self._ctx, _ptr(pts), pts.shape[0], _ptr(T_CW), _ptr(depth), F_, H, W,
                                               float(fx), float(fy), float(cx), float(cy), float(trunc), _ptr(vis),
                                               self._stream()))
        return vis

    def gt_sdf_grad(self, lattice, origin, spacing, pts, delta):
        """eval_pts.eval_grad(is_gt_sdf=True) on the lattice of gt_sdf_sample at pts [N,3] (float32 or float64): central
        differences of step delta, NaN where a lookup is outside the lattice or exactly 0.  Returns (grad fp64 [N,3],
        valid uint8 [N], 1 iff no component is NaN)."""
        lattice = self._arg(lattice, "lattice", F32, (None, None, None))
        pts = self._arg(pts, "pts", (F32, F64), (None, 3))
        grad = torch.empty(pts.shape[0], 3, dtype=torch.float64, device=self.device)
        valid = torch.empty(pts.shape[0], dtype=torch.uint8, device=self.device)
        self._ck(self.lib.isdfb_gt_sdf_grad(self._ctx, *self._lattice_args(lattice, origin, spacing, pts), float(delta),
                                            _ptr(grad), _ptr(valid), self._stream()))
        return grad, valid

    def sdf_split_stats(self, pred, gt, n_vox):
        """eval_pts.sub_eval's sums (device fp64 [2,17]): row 0 over all points, row 1 over the first n_vox, each in
        sdf_error_stats's layout, with no point left out."""
        n = pred.numel()
        pred, gt = self._arg(pred, "pred", F32, n), self._arg(gt, "gt", F64, n)
        if not 0 <= int(n_vox) <= n:
            raise ValueError("n_vox %d outside [0, %d]" % (n_vox, n))
        out = torch.empty(2, 17, dtype=torch.float64, device=self.device)
        self._ck(self.lib.isdfb_sdf_split_stats(self._ctx, _ptr(pred), _ptr(gt), n, int(n_vox), _ptr(out),
                                                self._stream()))
        return out

    def grad_cosdist(self, pred, gt, gt_index=None, eps=1e-6):
        """Sum over k of 1 - CosineSimilarity(dim=1, eps)(pred[k], gt[gt_index[k]]) (gt[k] without an index), in fp64
        (device tensor [1]).  pred fp32 [M,3], gt fp64 [N,3], gt_index int64 [M]."""
        pred = self._arg(pred, "pred", F32, (None, 3))
        m = pred.shape[0]
        gt_index = self._arg(gt_index, "gt_index", I64, m)
        gt = self._arg(gt, "gt", F64, (None if gt_index is not None else m, 3))
        out = torch.empty(1, dtype=torch.float64, device=self.device)
        self._ck(self.lib.isdfb_grad_cosdist(self._ctx, _ptr(pred), _ptr(gt), _ptr(gt_index), m, float(eps), _ptr(out),
                                             self._stream()))
        return out

    def chomp_costs(self, pred, gt, in_bounds, epsilons):
        """eval_traj_cost's sums (device fp64 [1 + 2 len(epsilons)]): the count of points in bounds with gt != 0, then
        per epsilon the sum of metrics.chomp_cost over their fp32 predictions, then the same over their fp64 GT."""
        n = pred.numel()
        pred, gt = self._arg(pred, "pred", F32, n), self._arg(gt, "gt", F64, n)
        in_bounds = self._arg(in_bounds, "in_bounds", U8, n)
        eps = [float(e) for e in epsilons]
        out = torch.empty(1 + 2 * len(eps), dtype=torch.float64, device=self.device)
        self._ck(self.lib.isdfb_chomp_costs(self._ctx, _ptr(pred), _ptr(gt), _ptr(in_bounds), n,
                                            (C.c_double * len(eps))(*eps), len(eps), _ptr(out), self._stream()))
        return out

    # ---- ground-truth SDF lattices from meshes ---------------------------
    def _mesh_args(self, verts, faces, pitch, origin):
        """The C arguments of isdfb_voxelize_count / _emit from the vertices to the origin."""
        verts = self._arg(verts, "verts", F64, (None, 3))
        faces = self._arg(faces, "faces", (I64, I32), (None, 3))
        org = (C.c_double * 3)(*[float(v) for v in origin])
        return (_ptr(verts), verts.shape[0], _ptr(faces), int(faces.dtype == I64), faces.shape[0], float(pitch), org), \
            (verts, faces)

    def voxelize(self, verts, faces, pitch, origin=(0., 0., 0.)):
        """voxelize_subdivide (sdf_util.py:312-368): the voxels rint((v - origin) / pitch) of every corner of the faces
        subdivided until no edge exceeds pitch / 2.  verts fp64 [V,3], faces int32 or int64 [F,3].  Returns (box_lo, a
        tuple of 3 ints: the smallest voxel index per axis; box uint8 [dx,dy,dz], 1 at the occupied voxels)."""
        args, keep = self._mesh_args(verts, faces, pitch, origin)
        lo, dims = (C.c_int64 * 3)(), (C.c_int64 * 3)()
        self._ck(self.lib.isdfb_voxelize_count(self._ctx, *args, lo, dims, self._stream()))
        box = torch.empty(tuple(dims), dtype=torch.uint8, device=self.device)
        self._ck(self.lib.isdfb_voxelize_emit(self._ctx, *args, lo, dims, _ptr(box), self._stream()))
        return tuple(lo), box

    def fill_holes(self, box):
        """scipy.ndimage.binary_fill_holes (6-connectivity) in place on the uint8 box [nx,ny,nz]; returns it (0 / 1)."""
        box = self._arg(box, "box", U8, (None, None, None), as_is=True)
        self._ck(self.lib.isdfb_fill_holes(self._ctx, _ptr(box), *box.shape, self._stream()))
        return box

    def occupancy_sdf(self, occ, voxel_size):
        """sdf_from_occupancy (sdf_util.py:371-385): (edt(occ == 0) - edt(occ != 0)) * voxel_size in fp64 [nx,ny,nz],
        bitwise scipy's; occ uint8 or bool [nx,ny,nz], neither all empty nor all occupied."""
        occ = self._arg(occ, "occ", U8, (None, None, None))
        sdf = torch.empty(occ.shape, dtype=torch.float64, device=self.device)
        self._ck(self.lib.isdfb_occupancy_sdf(self._ctx, _ptr(occ), *occ.shape, float(voxel_size), _ptr(sdf),
                                              self._stream()))
        return sdf

    # ---- N2 ----------------------------------------------------------
    def bounds_pc(self, pc, z_vals, depth_sample, ray_valid=None):
        """loss.bounds_pc (loss.py:56-89): bounds [R,S] and target directions [R,S,3] (row 0 unused)."""
        dev = self.device
        z_vals = self._arg(z_vals, "z_vals", F32, (None, None))
        R, S = z_vals.shape
        pc, depth_sample = self._arg(pc, "pc", F32, (R, S, 3)), self._arg(depth_sample, "depth_sample", F32, (R,))
        ray_valid = self._arg(ray_valid, "ray_valid", U8, (R,))
        bounds = torch.empty(R, S, dtype=torch.float32, device=dev)
        vec = torch.empty(R, S, 3, dtype=torch.float32, device=dev)
        self._ck(self.lib.isdfb_bounds_pc(self._ctx, _ptr(pc), _ptr(z_vals), _ptr(depth_sample), _ptr(ray_valid),
                                          R, S, _ptr(bounds), _ptr(vec), self._stream()))
        return bounds, vec

    # ---- K4 ----------------------------------------------------------
    def train_fwd_bwd(self, pc, z_vals, depth_sample, dirs_C, T_WC_sample, norm_sample, noise, loss_cfg,
                      ray_valid=None, want_grad=True, loss_sums=None):
        dev = self.device
        pc = self._arg(pc, "pc", F32, (None, None, 3))
        R, S = pc.shape[0], pc.shape[1]
        z_vals = self._arg(z_vals, "z_vals", F32, (R, S))
        depth_sample = self._arg(depth_sample, "depth_sample", F32, (R,))
        dirs_C = self._arg(dirs_C, "dirs_C_sample", F32, (R, 3))
        T_WC_sample = self._arg(T_WC_sample, "T_WC_sample", F32, (R, 4, 4))
        norm_sample = self._arg(norm_sample, "norm_sample", F32, (R, 3))
        noise, ray_valid = self._arg(noise, "noise", F32, (R, S)), self._arg(ray_valid, "ray_valid", U8, (R,))
        # the loss config already holds the raw addresses of its tensors: they are checked, never replaced
        self._arg(loss_cfg.bounds, "bounds", F32, (R, S), as_is=True)
        self._arg(loss_cfg.grad_vec, "grad_vec", F32, (R, S, 3), as_is=True)
        self._arg(loss_cfg.inv_count_tensor, "inv_count_dev", F32, (None,), rows=1, as_is=True)
        if loss_sums is None:
            loss_sums = torch.zeros(4, dtype=torch.float32, device=dev)
        loss_sums = self._arg(loss_sums, "loss_sums", F32, (4,), as_is=True)
        sdf = torch.empty(R, S, dtype=torch.float32, device=dev)
        g = torch.empty(R, S, 3, dtype=torch.float32, device=dev) if want_grad else None
        loss_mat = torch.empty(R, S, dtype=torch.float32, device=dev)
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
        out = self._arg(out, "out", F32, self.n_params, as_is=True)
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
        loss_mat = self._arg(loss_mat, "loss_mat", F32, (None, None))
        R, S = loss_mat.shape
        ib, ih, iw = (self._arg(ib, "indices_b", I64, (R,)), self._arg(ih, "indices_h", I64, (R,)),
                      self._arg(iw, "indices_w", I64, (R,)))
        ray_valid = self._arg(ray_valid, "ray_valid", U8, (R,))
        approx = torch.empty(n_frames, factor, factor, dtype=torch.float32, device=dev)
        favg = torch.empty(n_frames, dtype=torch.float32, device=dev)
        self._ck(self.lib.isdfb_frame_bins(self._ctx, _ptr(loss_mat), _ptr(ray_valid), _ptr(ib), _ptr(ih), _ptr(iw),
                                           R, S, int(n_frames), int(H), int(W), int(factor), _ptr(approx),
                                           _ptr(favg), self._stream()))
        return approx, favg

    def step_finish(self, loss_mat, ib, ih, iw, n_frames, H, W, factor, ray_valid, frame_map, frame_avg_losses,
                    loss_sums, inv_count, means_out):
        """K5 + write-back of the per-keyframe losses + the four loss means (clears loss_sums); see the header.  It runs
        inside the captured step, and takes its tensors as they are: only ray_valid may be converted."""
        dev = self.device
        loss_mat = self._arg(loss_mat, "loss_mat", F32, (None, None), as_is=True)
        R, S = loss_mat.shape
        ib = self._arg(ib, "indices_b", I64, (R,), as_is=True)
        ih, iw = self._arg(ih, "indices_h", I64, (R,), as_is=True), self._arg(iw, "indices_w", I64, (R,), as_is=True)
        ray_valid = self._arg(ray_valid, "ray_valid", U8, (R,))
        frame_map = self._arg(frame_map, "frame_map", I64, (None,), rows=n_frames, as_is=True)
        frame_avg_losses = self._arg(frame_avg_losses, "frame_avg_losses", F32, (None,), rows=n_frames, as_is=True)
        loss_sums = self._arg(loss_sums, "loss_sums", F32, (4,), as_is=True)
        inv_count = self._arg(inv_count, "inv_count", F32, (None,), rows=1, as_is=True)
        means_out = self._arg(means_out, "means_out", F32, (4,), as_is=True)
        approx = torch.empty(n_frames, factor, factor, dtype=torch.float32, device=dev)
        favg = torch.empty(n_frames, dtype=torch.float32, device=dev)
        self._ck(self.lib.isdfb_step_finish(self._ctx, _ptr(loss_mat), _ptr(ray_valid), _ptr(ib), _ptr(ih), _ptr(iw), R, S,
                                            int(n_frames), int(H), int(W), int(factor), _ptr(approx), _ptr(favg),
                                            _ptr(frame_map), _ptr(frame_avg_losses), _ptr(loss_sums), _ptr(inv_count),
                                            _ptr(means_out), self._stream()))
        return approx, favg

    def select_window(self, frame_avg_losses, n_frames, window_size, seed, out=None):
        """A0 on the device: Gumbel top-k window (see isdfb_select_window)."""
        w = self._arg(frame_avg_losses, "frame_avg_losses", F32, (None,), rows=n_frames)
        if out is None:
            out = torch.empty(window_size, dtype=torch.int64, device=self.device)
        out = self._arg(out, "out", I64, (window_size,), as_is=True)
        self._ck(self.lib.isdfb_select_window(self._ctx, _ptr(w), int(n_frames), int(window_size),
                                              C.c_uint64(int(seed) & (2 ** 64 - 1)), _ptr(out), self._stream()))
        return out

    # ---- K6 ----------------------------------------------------------
    def _adamw_state(self, params, m, v):
        n = self.n_params
        return (_ptr(self._arg(params, "params", F32, n, as_is=True)),
                _ptr(self._arg(m, "exp_avg", F32, n, as_is=True)), _ptr(self._arg(v, "exp_avg_sq", F32, n, as_is=True)))

    def adamw(self, params, m, v, step, lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01, grad_scale=1.0):
        self._ck(self.lib.isdfb_adamw(self._ctx, *self._adamw_state(params, m, v), int(step), float(lr), float(beta1),
                                      float(beta2), float(eps), float(weight_decay), float(grad_scale),
                                      self._stream()))

    def adamw_graph(self, params, m, v, lr, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.01, grad_scale=1.0):
        """K6 with the step counter on the device (CUDA-graph capturable)."""
        self._ck(self.lib.isdfb_adamw_graph(self._ctx, *self._adamw_state(params, m, v), float(lr), float(beta1),
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

    # ---- debug hook ------------------------------------------------------
    def debug_buffers(self):
        """isdfb_debug_buffers: the tensor-core path's raw per-tile side arrays as device addresses (0: absent) with
        their strides and counts (see the header)."""
        aux, dhi, dlo, sg = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
        a_st, d_st, tiles = C.c_int64(), C.c_int64(), C.c_int64()
        n_aux, n_dwl = C.c_int32(), C.c_int32()
        self._ck(self.lib.isdfb_debug_buffers(self._ctx, C.byref(aux), C.byref(a_st), C.byref(dhi), C.byref(dlo),
                                              C.byref(d_st), C.byref(n_aux), C.byref(n_dwl), C.byref(tiles), C.byref(sg)))
        return dict(aux=aux.value or 0, aux_stride_floats=a_st.value, dwl_hi=dhi.value or 0, dwl_lo=dlo.value or 0,
                    dwl_stride_bytes=d_st.value, n_aux=n_aux.value, n_dwl=n_dwl.value, tiles=tiles.value,
                    sig16=sg.value or 0)


class _DevView:
    """Wrap a raw device pointer as a torch tensor through __cuda_array_interface__."""

    def __init__(self, ptr, n, device):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (ptr, False), "version": 2}
        self.tensor = torch.as_tensor(self, device=device)


def make_loss_cfg(trunc_weight, trunc_distance, eik_weight, eik_apply_dist, grad_weight, orien_loss, loss_type,
                  noise_std, inv_count, inv_count_dev=None, bounds=None, grad_vec=None):
    """The loss config of Engine.train_fwd_bwd, which checks the tensors it keeps against the batch."""
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
    if (bounds is None) != (grad_vec is None):
        raise ValueError("bounds and grad_vec (the outputs of Engine.bounds_pc) go together")
    # the struct holds raw addresses: the tensors stay referenced by the config
    lc.inv_count_tensor, lc.bounds, lc.grad_vec = inv_count_dev, bounds, grad_vec
    lc.inv_count_dev, lc.bounds_dev, lc.grad_vec_dev = [None if t is None else t.data_ptr()
                                                        for t in (inv_count_dev, bounds, grad_vec)]
    return lc


def make_camera(fx, fy, cx, cy, H, W):
    cam = _lib.Camera()
    cam.fx, cam.fy, cam.cx, cam.cy, cam.H, cam.W = float(fx), float(fy), float(cx), float(cy), int(H), int(W)
    return cam


def pe_nat_col(c, half):
    """Internal embedding column -> the reference's column (tc_common.cuh pe_nat_col): [sin_0 cos_0 sin_1 cos_1 ... |
    x y z | pad] -> [x y z | sin(xb) | sin(xb + pi/2)]; `half` = 21 n_freqs."""
    if half <= 0:
        return c
    if c < 2 * half:
        return 3 + (c >> 1) + (c & 1) * half
    if c < 2 * half + 3:
        return c - 2 * half
    return c


class SideState:
    """Test helper: the tensor-core path's per-tile side state of the LAST chunk it ran, decoded on the device into
    [points, columns] fp32 tensors.  The array indices are those of tc_create (csrc/tc_path.cu), the element layouts
    those the chain kernel writes through off_a / off_d / off_x (csrc/tc_chain.cu, tc_common.cuh):

      aux   fp32 [f/4][128 points][4]:     partial sums 0 .. n_part-1 (3; 6 with two embedding halves), e32 per half,
                                          h_last, and (strict modes only) zbar2_l for every layer l
      dW    bf16 [p/16][f/8][16 points][8]: yh_l (0 .. L-1: e, h_0 .. h_{L-2}), ya_l (L ..: abar_e, abar_0 ..),
                                          xd_l = delta_l, xz_l = zbar_l, v, and with two halves yh_e1, ya_e1;
                                          hi image always, lo image in bf16x3 only
      sig16 unorm16 [f/8][128 points][8]: sigma_l for every layer l; in bf16x3g the bf16 zbar2_l image follows at
                                          layer L + l (same layout)

    Embedding-fed arrays (e32, yh_0, ya_0 and the second half's) hold the internal column order; `natural` maps them to
    the reference's.  Rows past the batch's last point are the padded rows of the last tile."""

    def __init__(self, engine, n_points):
        b = engine.debug_buffers()
        self.L = 2 * engine.block + 2
        self.E = engine.embedding_size
        self.NE = 2 if self.E > 256 else 1
        self.half = 21 * engine.n_freqs
        self.lean = engine.precision == "bf16x3g"
        self.n = int(n_points)
        self.tiles = -(-self.n // 128)
        self.rows = 128 * self.tiles
        cap, d_st, L, NE = b["tiles"], b["dwl_stride_bytes"], self.L, self.NE
        n_part = 6 if NE == 2 else 3
        # tc_create's indices
        self.arr_part, self.arr_e32, self.arr_hlast, self.arr_zb2 = 0, n_part, n_part + NE, n_part + NE + 1
        self.arr_yh, self.arr_ya, self.arr_xd, self.arr_xz, self.arr_v = 0, L, 2 * L, 3 * L, 4 * L
        self.arr_yh_e1, self.arr_ya_e1 = 4 * L + 1, 4 * L + 2
        assert b["n_aux"] == n_part + NE + 1 + (0 if self.lean else L), b
        assert b["n_dwl"] == 4 * L + 1 + (2 if NE == 2 else 0), b
        assert self.tiles <= cap
        dev = engine.device
        self._engine = engine                      # the views below are the context's memory: keep it alive
        self.has_lo = bool(b["dwl_lo"])
        self._aux = _DevView(b["aux"], b["aux_stride_floats"] * b["n_aux"], dev).tensor.view(b["n_aux"], cap, 64, 128, 4)

        def bytes16(ptr, n_arr):
            return _DevView(ptr, d_st * n_arr // 4, dev).tensor.view(torch.int16)

        self._hi = bytes16(b["dwl_hi"], b["n_dwl"]).view(b["n_dwl"], cap, 8, 32, 16, 8)
        self._lo = bytes16(b["dwl_lo"], b["n_dwl"]).view(b["n_dwl"], cap, 8, 32, 16, 8) if b["dwl_lo"] else None
        n_sig = L * (2 if self.lean else 1)
        self._sig = bytes16(b["sig16"], n_sig).view(n_sig, cap, 32, 128, 8)
        idx = [pe_nat_col(c, self.half) for c in range(256 * NE)]
        self._nat_src = torch.tensor([c for c in range(256 * NE) if idx[c] < self.E], device=dev)
        self._nat_dst = torch.tensor([idx[c] for c in range(256 * NE) if idx[c] < self.E], device=dev)

    # ---- raw arrays, [tiles * 128, 256], internal column order ----
    def aux(self, arr):
        return self._aux[arr, :self.tiles].permute(0, 2, 1, 3).reshape(self.rows, 256).clone()

    def dwl(self, arr, part="hi"):
        """One dW-layout array: part 'hi' or 'lo' (bf16x3 only) as fp32."""
        src = self._hi if part == "hi" else self._lo
        if src is None:
            raise ValueError("no %s image in %s mode" % (part, "bf16x3g" if self.lean else "this"))
        x = src[arr, :self.tiles].permute(0, 1, 3, 2, 4).reshape(self.rows, 256).contiguous()
        return x.view(torch.bfloat16).float()

    def sigma_code(self, l):
        """sigma_l as its unorm16 code (0 .. 65535, int32)."""
        return self._sig[l, :self.tiles].permute(0, 2, 1, 3).reshape(self.rows, 256).to(torch.int32) & 0xFFFF

    def sigma(self, l):
        return self.sigma_code(l).float() / 65535.0

    def zbar2(self, l):
        """zbar2_l: fp32 side array (bf16x3, bf16) or the bf16 image behind sigma (bf16x3g)."""
        if not self.lean:
            return self.aux(self.arr_zb2 + l)
        x = self._sig[self.L + l, :self.tiles].permute(0, 2, 1, 3).reshape(self.rows, 256).contiguous()
        return x.view(torch.bfloat16).float()

    # ---- embedding-fed arrays ----
    def natural(self, halves):
        """Internal columns of the embedding halves (list of [rows, 256]) -> [rows, E] in the reference's order."""
        x = torch.cat(halves, dim=1)
        out = torch.zeros(x.shape[0], self.E, dtype=x.dtype, device=x.device)
        out[:, self._nat_dst] = x[:, self._nat_src]
        return out

    def e32(self):
        """The fp32 embedding, [rows, E] natural order."""
        return self.natural([self.aux(self.arr_e32 + h) for h in range(self.NE)])

    def operand(self, name, l=0, part="hi"):
        """A weight-gradient operand by name: 'yh' (l = 0: e, l >= 1: h_{l-1}), 'ya' (l = 0: abar_e, l >= 1:
        abar_{l-1}), 'xd' (delta_l), 'xz' (zbar_l), 'v'.  yh_0 and ya_0 come back as [rows, E] in natural order."""
        if name == "v":
            return self.dwl(self.arr_v, part)
        base = dict(yh=self.arr_yh, ya=self.arr_ya, xd=self.arr_xd, xz=self.arr_xz)[name]
        if name in ("yh", "ya") and l == 0:
            halves = [self.dwl(base, part)]
            if self.NE == 2:
                halves.append(self.dwl(self.arr_yh_e1 if name == "yh" else self.arr_ya_e1, part))
            return self.natural(halves)
        return self.dwl(base + l, part)


def debug_state(engine, n_points):
    """Test helper: the decoded side state of the last chunk (see SideState)."""
    return SideState(engine, n_points)
