"""Ground-truth SDF lattices from meshes on the GPU -- mirror of sdf_from_occupancy, sdf_from_mesh and
sdf_from_mesh_gridgiven of the reference's isdf/datasets/sdf_util.py (:371-457).

Same signatures and return types as the reference (numpy float64 `sdf`, 4x4 `transform`); the voxelization
(voxelize_subdivide), the hole fill (VoxelGrid.fill) and the distance transforms run in the CUDA kernels behind
Engine.voxelize / fill_holes / occupancy_sdf on the current CUDA device.  The index arithmetic that places the object
into the lattice is the reference's, on the host.  Every other name of the reference module (read_sdf_*, merge_sdfs,
the colormaps, ...) is served by the reference's own file through the `isdf` alias.  Neither trimesh nor matplotlib is
imported: a mesh is anything with `vertices` [V,3] and `faces` [F,3]."""
import numpy as np
import torch

from .. import _lib
from ..engine import Engine

_ENGINES = {}


def _engine():
    """A small context of the current CUDA device (the model-shaped part is the smallest the library takes)."""
    if not torch.cuda.is_available():
        raise RuntimeError("isdf_b200.datasets.sdf_util runs on a CUDA device; there is no CPU path")
    index = torch.cuda.current_device()
    if index not in _ENGINES:
        _ENGINES[index] = Engine(torch.device("cuda", index), 1, 128, 1, 1.0, 1.0, precision="fp32", max_points=128)
    return _ENGINES[index]


def _refusal(fn, *args):
    """An argument or capacity refusal of a C entry as ValueError, as the reference's numpy / trimesh would raise."""
    try:
        return fn(*args)
    except _lib.IsdfbError as e:
        if e.rc in (_lib.ERR_ARG, _lib.ERR_CAPACITY):
            raise ValueError(str(e)) from e
        raise


def _occupied_box(mesh, pitch, origin_voxel):
    """voxelize_subdivide(mesh, pitch, origin_voxel).fill(): (.matrix as a device uint8 box, .transform)."""
    eng = _engine()
    verts = torch.as_tensor(np.ascontiguousarray(np.asarray(mesh.vertices, dtype=np.float64).reshape(-1, 3)),
                            device=eng.device)
    faces = np.asarray(mesh.faces).reshape(-1, 3)
    faces = torch.as_tensor(np.ascontiguousarray(faces if faces.dtype in (np.int32, np.int64) else faces.astype(np.int64)),
                            device=eng.device)
    origin_voxel = np.asarray(origin_voxel, dtype=np.float64)
    lo, box = _refusal(eng.voxelize, verts, faces, float(pitch), origin_voxel.tolist())
    eng.fill_holes(box)
    # trimesh.transformations.scale_and_translate(scale=pitch, translate=origin_voxel + origin_index * pitch)
    transform = np.eye(4)
    transform[:3, :3] *= pitch
    transform[:3, 3] = origin_voxel + np.array(lo, dtype=np.int64) * pitch
    return box, transform


def _sdf(occ, voxel_size):
    """(edt(~occ) - edt(occ)) * voxel_size of the device uint8 lattice occ, as a numpy float64 array."""
    if min(occ.shape) < 1:
        raise ValueError("occupancy lattice %s has an empty axis" % (tuple(occ.shape),))
    return _refusal(_engine().occupancy_sdf, occ, float(voxel_size)).cpu().numpy()


def sdf_from_occupancy(occ_map, voxel_size):
    """sdf_util.sdf_from_occupancy: signed distance in metric units, positive in free space, from a boolean (or 0 / 1)
    occupancy map [nx,ny,nz].  Refused (ValueError): a map that is all empty or all occupied (scipy's transform has
    no feature to measure to), an empty axis, and values other than 0 and 1."""
    occ = np.asarray(occ_map)
    if occ.ndim != 3:
        raise ValueError("occupancy map must be 3-D, got shape %s" % (occ.shape,))
    if occ.dtype != np.bool_:
        if not np.isin(occ, (0, 1)).all():
            raise ValueError("occupancy map must hold only 0 and 1")
        occ = occ != 0
    return _sdf(torch.as_tensor(np.ascontiguousarray(occ.astype(np.uint8)), device=_engine().device), voxel_size)


def sdf_from_mesh(mesh, voxel_size, extend_factor=0.15, origin_voxel=np.zeros(3)):
    """sdf_util.sdf_from_mesh: the SDF of the mesh on its own voxel box, padded by round(shape * extend_factor) voxels
    on every side.  Returns (sdf float64 [nx,ny,nz], transform 4x4 with the voxel size on the diagonal and the first
    voxel's centre as translation)."""
    box, transform = _occupied_box(mesh, voxel_size, origin_voxel)
    extend = np.array(box.shape) * extend_factor
    extend = np.repeat(extend, 2).reshape(3, 2)
    extend = np.round(extend).astype(int)
    occ = torch.zeros(tuple(int(s) + int(e[0]) + int(e[1]) for s, e in zip(box.shape, extend)), dtype=torch.uint8,
                      device=box.device)
    occ[extend[0, 0]:extend[0, 0] + box.shape[0], extend[1, 0]:extend[1, 0] + box.shape[1],
        extend[2, 0]:extend[2, 0] + box.shape[2]] = box
    transform[:3, 3] -= extend[:, 0] * voxel_size
    return _sdf(occ, voxel_size), transform


def sdf_from_mesh_gridgiven(mesh, transform, dims):
    """sdf_util.sdf_from_mesh_gridgiven: the SDF of the mesh in the lattice of `dims` voxels whose first voxel centre
    and voxel size the 4x4 `transform` gives; the part of the object outside the lattice is cropped.  Returns (sdf
    float64 [dims], transform).  AssertionError "Grids are not aligned" as the reference; ValueError for an object that
    leaves the lattice empty."""
    voxel_size = transform[0, 0]
    origin_voxel = transform[:3, 3] % transform[0, 0]
    occ_map, occ_transform = _occupied_box(mesh, voxel_size, origin_voxel)
    dims = tuple(int(d) for d in dims)
    if len(dims) != 3 or min(dims) < 1:
        raise ValueError("dims must be three positive sizes, got %s" % (dims,))

    # the reference's index arithmetic (sdf_util.py:424-442), on the host
    base_shape = np.array(dims)
    base_start_ix = (occ_transform[:3, 3] - transform[:3, 3]) / voxel_size
    base_end_ix = base_start_ix + occ_map.shape

    check = base_start_ix - np.round(base_start_ix)
    if not np.linalg.norm(check) < 1e-5:
        raise AssertionError("Grids are not aligned")

    occ_start_ix = np.maximum(np.zeros_like(base_start_ix), -base_start_ix)
    occ_end_ix = base_shape - base_end_ix
    coords = np.argwhere(occ_end_ix >= 0)
    occ_end_ix[coords] = np.array(occ_map.shape)[coords]

    base_end_ix = np.minimum(base_shape, base_end_ix)
    base_start_ix[base_start_ix < 0] = 0

    base_start_ix = np.round(base_start_ix).astype(int)
    base_end_ix = np.round(base_end_ix).astype(int)
    occ_start_ix = np.round(occ_start_ix).astype(int)
    occ_end_ix = np.round(occ_end_ix).astype(int)

    base_grid = torch.zeros(dims, dtype=torch.uint8, device=occ_map.device)
    occ_inrange = occ_map[occ_start_ix[0]:occ_end_ix[0], occ_start_ix[1]:occ_end_ix[1], occ_start_ix[2]:occ_end_ix[2]]
    target = base_grid[base_start_ix[0]:base_end_ix[0], base_start_ix[1]:base_end_ix[1],
                       base_start_ix[2]:base_end_ix[2]]
    if tuple(target.shape) != tuple(occ_inrange.shape):
        raise ValueError("could not place the object's box %s into the lattice slice %s"
                         % (tuple(occ_inrange.shape), tuple(target.shape)))
    target.copy_(occ_inrange)
    return _sdf(base_grid, voxel_size), transform
