"""Posed-depth sources for the Trainer.

`SyntheticStream` is the seeded synthetic stream of SURVEY.md 8d (the real sequences are not
available offline); `ReplicaDataset` reads the reference's ReplicaCAD on-disk layout
(reference isdf/datasets/dataset.py:20-71: results/depth%06d.png, frame%06d.png, traj.txt), `ScanNetDataset` its ScanNet
layout and `RealsenseFrankaOffline` its recorded Franka tabletop sequences."""
import math
import os

import numpy as np


class SyntheticStream:
    """Frame k: depth[v,u] = 2 + 0.5 sin(u/80 + 0.1k) + 0.3 cos(v/60) metres, small yaw + translation."""

    def __init__(self, n_frames, H, W, invalid_frac=0.0, seed=1234, depth_scale=1000.0, rot=True):
        self.n_frames, self.H, self.W = n_frames, H, W
        self.invalid_frac, self.seed, self.depth_scale, self.rot = invalid_frac, seed, depth_scale, rot
        v = np.arange(H, dtype=np.float32)[:, None]
        u = np.arange(W, dtype=np.float32)[None, :]
        self._v_term = (0.3 * np.cos(v / 60.0)).astype(np.float32)
        self._u = u
        self.cache_frames = False          # True: keep generated host frames (they stand in for decoded images)
        self._cache = {}

    def __len__(self):
        return self.n_frames

    def pose(self, k):
        T = np.eye(4, dtype=np.float32)
        if self.rot:
            a = 0.05 * k
            c, s = math.cos(a), math.sin(a)
            T[0, 0], T[0, 2], T[2, 0], T[2, 2] = c, s, -s, c
        T[0, 3], T[1, 3] = 0.05 * k, 0.01 * k
        return T

    def depth(self, k):
        d = (2.0 + 0.5 * np.sin(self._u / 80.0 + 0.1 * k) + self._v_term).astype(np.float32)
        if self.invalid_frac > 0:
            rng = np.random.default_rng(self.seed + k)
            d[rng.random((self.H, self.W)) < self.invalid_frac] = 0.0
        return d

    def __getitem__(self, k):
        k = int(k) % self.n_frames
        if k in self._cache:
            return self._cache[k]
        image = np.full((self.H, self.W, 3), 128, dtype=np.uint8)
        item = {"image": image, "depth": self.depth(k), "T": self.pose(k)}
        if self.cache_frames:
            # cached frames stand in for decoded camera images waiting in a capture queue: kept in page-locked memory, so
            # Trainer.get_data can copy them to the device without a staging pass ("depth_pinned" aliases "depth")
            try:
                import torch
                if torch.cuda.is_available():
                    pin = torch.from_numpy(item["depth"]).pin_memory()
                    item["depth_pinned"] = pin
                    item["depth"] = pin.numpy()
            except Exception:      # noqa: BLE001 -- pinning is an optimisation only
                pass
            self._cache[k] = item
        return item


class ReplicaDataset:
    def __init__(self, root_dir, traj_file=None, rgb_transform=None, depth_transform=None, noisy_depth=False,
                 col_ext=".jpg", distortion_coeffs=None, camera_matrix=None):
        self.Ts = None if traj_file is None else np.loadtxt(traj_file).reshape(-1, 4, 4)
        self.root_dir = root_dir
        self.rgb_transform, self.depth_transform = rgb_transform, depth_transform
        self.col_ext, self.noisy_depth = col_ext, noisy_depth

    def __len__(self):
        return self.Ts.shape[0]

    def __getitem__(self, idx):
        import cv2
        s = "%06d" % int(idx)
        depth_file = os.path.join(self.root_dir, ("ndepth" if self.noisy_depth else "depth") + s + ".png")
        rgb_file = os.path.join(self.root_dir, "frame" + s + self.col_ext)
        depth = cv2.imread(depth_file, -1)
        image = cv2.imread(rgb_file)
        if depth is None or image is None:
            raise FileNotFoundError("missing frame %s under %s" % (s, self.root_dir))
        T = self.Ts[idx] if self.Ts is not None else None
        if self.rgb_transform:
            image = self.rgb_transform(image)
        if self.depth_transform:
            depth = self.depth_transform(depth)
        return {"image": image, "depth": depth, "T": T}


class ScanNetDataset:
    """ScanNet layout of the reference (datasets/dataset.py:74-121): <root>/frames/color/<i>.jpg,
    <root>/frames/depth/<i>.png (uint16), poses as N x 16 rows in `traj_file`."""

    def __init__(self, root_dir, traj_file, rgb_transform=None, depth_transform=None, col_ext=".jpg",
                 noisy_depth=None, distortion_coeffs=None, camera_matrix=None):
        self.root_dir = root_dir
        self.rgb_dir = os.path.join(root_dir, "frames", "color")
        self.depth_dir = os.path.join(root_dir, "frames", "depth")
        self.Ts = None if traj_file is None else np.loadtxt(traj_file).reshape(-1, 4, 4)
        self.rgb_transform, self.depth_transform, self.col_ext = rgb_transform, depth_transform, col_ext or ".jpg"

    def __len__(self):
        return self.Ts.shape[0]

    def __getitem__(self, idx):
        import cv2
        idx = int(idx)
        depth = cv2.imread(os.path.join(self.depth_dir, "%d.png" % idx), -1)
        image = cv2.imread(os.path.join(self.rgb_dir, "%d%s" % (idx, self.col_ext)))
        if depth is None or image is None:
            raise FileNotFoundError("missing ScanNet frame %d under %s" % (idx, self.root_dir))
        T = self.Ts[idx] if self.Ts is not None else None
        if self.rgb_transform:
            image = self.rgb_transform(image)
        if self.depth_transform:
            depth = self.depth_transform(depth)
        return {"image": image, "depth": depth, "T": T}


class RealsenseFrankaOffline:
    """Recorded Franka tabletop sequences of the reference (datasets/dataset.py:123-173): <root>/depth/%05d.npy (uint16
    millimetres as the recorder writes them), <root>/rgb/%05d<col_ext>, and `traj_file` rows of a timestamp followed by
    the 16 entries of the pose.  Unlike the reference the constructor does not change the process's working directory:
    a relative `root_dir` or `traj_file` is resolved against the current directory, as for the other readers."""

    def __init__(self, root_dir, traj_file, rgb_transform=None, depth_transform=None, col_ext=".jpg",
                 noisy_depth=None, distortion_coeffs=None, camera_matrix=None):
        if traj_file is None:
            raise ValueError("RealsenseFrankaOffline needs traj_file: the recorded poses (timestamp + 16 values per row) "
                             "are the only source of the camera poses")
        self.root_dir = root_dir
        self.rgb_dir = os.path.join(root_dir, "rgb")
        self.depth_dir = os.path.join(root_dir, "depth")
        self.Ts = np.loadtxt(traj_file, ndmin=2)[:, 1:].reshape(-1, 4, 4)
        self.rgb_transform, self.depth_transform, self.col_ext = rgb_transform, depth_transform, col_ext or ".jpg"

    def __len__(self):
        return self.Ts.shape[0]

    def __getitem__(self, idx):
        import cv2
        idx = int(idx)
        s = "%05d" % idx
        depth_file = os.path.join(self.depth_dir, s + ".npy")
        if not os.path.isfile(depth_file):
            raise FileNotFoundError("missing Franka depth frame %s" % depth_file)
        depth = np.load(depth_file)
        image = cv2.imread(os.path.join(self.rgb_dir, s + self.col_ext))
        if image is None:
            raise FileNotFoundError("missing Franka frame %s under %s" % (s + self.col_ext, self.rgb_dir))
        T = self.Ts[idx]
        if self.rgb_transform:
            image = self.rgb_transform(image)
        if self.depth_transform:
            depth = self.depth_transform(depth)
        return {"image": image, "depth": depth, "T": T}


def read_scannet_intrinsics(file):
    """fx, fy, cx, cy, H, W of the DEPTH camera from a ScanNet scene .txt (trainer.py:335-346)."""
    info = dict(line.split(' = ') for line in open(file).read().splitlines() if ' = ' in line)
    return (float(info['fx_depth']), float(info['fy_depth']), float(info['mx_depth']), float(info['my_depth']),
            int(info['depthHeight']), int(info['depthWidth']))


def depth_scale_filter(inv_scale, max_depth):
    """uint16 depth -> metres, far values zeroed (reference datasets/image_transforms.py:18-38)."""
    def f(depth):
        d = depth.astype(np.float32) * inv_scale
        d[d > max_depth] = 0.0
        return d
    return f


def bgr_to_rgb(image):
    return image[:, :, ::-1].copy()
