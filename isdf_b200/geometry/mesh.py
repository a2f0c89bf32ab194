"""The triangle mesh Trainer.mesh_rec returns and its PLY writer (the parts of trimesh the reference's mesh_rec /
write_mesh use, trainer.py:1500-1556)."""
import numpy as np

# draw3D.draw_mesh(color_by="none") paints every face this colour (draw3D.py:157-158)
FACE_RGBA = (160, 160, 160, 255)


class Mesh:
    """vertices [V,3] float64, faces [F,3] int64 (indices into vertices)."""

    def __init__(self, vertices, faces):
        self.vertices = np.ascontiguousarray(vertices, dtype=np.float64).reshape(-1, 3)
        self.faces = np.ascontiguousarray(faces, dtype=np.int64).reshape(-1, 3)

    def __repr__(self):
        return "Mesh(vertices=%d, faces=%d)" % (len(self.vertices), len(self.faces))


def export_ply(mesh, face_rgba=FACE_RGBA):
    """Binary little-endian PLY: float32 x y z per vertex; per face `list uchar int vertex_indices` and an
    uchar red green blue alpha colour (what trimesh.exchange.ply.export_ply writes for a face-coloured mesh, without
    aiming at byte equality)."""
    v = np.asarray(mesh.vertices, dtype="<f4").reshape(-1, 3)
    f = np.asarray(mesh.faces).reshape(-1, 3)
    if len(f) and (f.min() < 0 or f.max() >= len(v)):
        raise ValueError("face index outside the vertex array")
    header = ("ply\nformat binary_little_endian 1.0\n"
              "element vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
              "element face %d\nproperty list uchar int vertex_indices\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\nproperty uchar alpha\n"
              "end_header\n" % (len(v), len(f)))
    rec = np.zeros(len(f), dtype=np.dtype([("n", "u1"), ("v", "<i4", (3,)), ("rgba", "u1", (4,))]))
    rec["n"] = 3
    rec["v"] = f
    rec["rgba"] = face_rgba
    return header.encode("ascii") + v.tobytes() + rec.tobytes()
