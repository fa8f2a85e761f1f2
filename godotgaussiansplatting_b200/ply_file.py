"""Host-side mirror of the reference's `PlyFile` resource (util/ply_file.gd).

`PlyFile.parse` follows util/ply_file.gd:10-19 (header scan, whole body as one float32 array) and
`load_gaussian_splats` follows util/ply_file.gd:28-77: per splat exp(scale), quaternion -> rotation,
Sigma = R S^2 R^T (upper triangle), sigmoid(opacity) and the SH re-interleave into the 60-float
std430 `Splat` struct (gsplat_projection.glsl:33-40) -- vectorised numpy instead of a GDScript loop,
then chunked uploads through the C-ABI (`gsr_upload_splats_aos`), mirroring the ~1000 chunked
`buffer_update`s of the reference.  In the reference this step also runs on the host CPU.

All float32 operations are written one IEEE op at a time in the order Godot's `Basis`/`Quaternion`
code evaluates them, so the result is bit-identical to the C oracle's restatement (tests/test_oracle.py).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

STRUCT_SIZE = 60  # floats (util/ply_file.gd:29)
F = np.float32


class PlyFile:
    """util/ply_file.gd:1-26.  Attributes: size, vertices (flat float32), properties (names)."""

    def __init__(self, path: str = ""):
        self.size = 0
        self.vertices = np.zeros(0, dtype=np.float32)
        self.properties: list[str] = []
        if path:
            self.parse(path)

    @classmethod
    def from_array(cls, vertices: np.ndarray, properties: list[str] | None = None) -> "PlyFile":
        """Build a PlyFile from an (n, nprops) float32 array (synthetic scenes)."""
        v = np.ascontiguousarray(vertices, dtype=np.float32)
        self = cls()
        self.size = int(v.shape[0])
        self.properties = list(properties) if properties is not None else default_properties(v.shape[1])
        self.vertices = v.reshape(-1)
        return self

    def parse(self, path: str) -> None:  # util/ply_file.gd:10-19
        big_endian = False
        with open(path, "rb") as f:
            while True:
                raw = f.readline()
                if not raw:
                    raise ValueError("PLY header has no end_header")
                line = raw.decode("ascii", "replace").strip().split(" ")
                if line[0] == "end_header":
                    break
                if line[0] == "format":
                    big_endian = line[1] == "binary_big_endian"
                elif line[0] == "element":
                    self.size = int(line[2])
                elif line[0] == "property":
                    self.properties.append(line[2])
            count = self.size * len(self.properties)
            body = np.fromfile(f, dtype=">f4" if big_endian else "<f4", count=count)
        if body.size != count:
            raise ValueError(f"PLY body truncated: {body.size} of {count} floats")
        self.vertices = body.astype(np.float32, copy=False)

    def get_vertex(self, index: int) -> dict:  # util/ply_file.gd:21-26
        n = len(self.properties)
        return {self.properties[i]: float(self.vertices[n * index + i]) for i in range(n)}

    @property
    def table(self) -> np.ndarray:
        return self.vertices.reshape(self.size, len(self.properties))

    def layout(self) -> "PlyLayout":
        """Where each property group sits in a vertex, and the file's SH degree, from the property names (include/gsr.h
        gsr_ply_layout).  Normals and extra properties are allowed anywhere; every group must be contiguous and in order."""
        names = list(self.properties)
        pos = {n: i for i, n in enumerate(names)}

        def group(first_names):
            missing = [n for n in first_names if n not in pos]
            if missing:
                raise ValueError(f"PLY has no {', '.join(missing)} property")
            at = pos[first_names[0]]
            if [pos[n] for n in first_names] != list(range(at, at + len(first_names))):
                raise ValueError(f"PLY properties {first_names[0]}..{first_names[-1]} are not contiguous")
            return at

        n_rest = sum(1 for n in names if n.startswith("f_rest_"))
        if n_rest not in SH_REST_FLOATS:
            raise ValueError(f"PLY has {n_rest} f_rest properties; an SH degree 0..3 file has 0, 9, 24 or 45")
        degree = SH_REST_FLOATS.index(n_rest)
        return PlyLayout(nprops=len(names), sh_degree=degree, x=group(["x", "y", "z"]), f_dc=group([f"f_dc_{i}" for i in range(3)]),
                         f_rest=group([f"f_rest_{i}" for i in range(n_rest)]) if n_rest else -1, opacity=group(["opacity"]),
                         scale=group([f"scale_{i}" for i in range(3)]), rot=group([f"rot_{i}" for i in range(4)]),
                         filter_3d=pos.get("filter_3D", -1))


SH_REST_FLOATS = (0, 9, 24, 45)   # f_rest floats of an SH degree 0..3 file: 3 * ((degree + 1)^2 - 1)


@dataclass(frozen=True)
class PlyLayout:
    """include/gsr.h gsr_ply_layout: index of x (y, z follow), f_dc_0, f_rest_0 (-1 iff degree 0), opacity, scale_0, rot_0; and
    filter_3d, the index of Mip-Splatting's `filter_3D` property or -1 (the filter_3d argument of gsr_upload_ply_filtered)."""
    nprops: int
    sh_degree: int
    x: int
    f_dc: int
    f_rest: int
    opacity: int
    scale: int
    rot: int
    filter_3d: int = -1


PLY_LAYOUT_3DGS = PlyLayout(nprops=62, sh_degree=3, x=0, f_dc=6, f_rest=9, opacity=54, scale=55, rot=58)   # the original 3DGS trainer's


def degree_properties(sh_degree: int, normals: bool = True, extra: tuple = ()) -> list[str]:
    """Property names of a 3DGS PLY of SH degree `sh_degree` (the trainer's order), optionally without nx ny nz, plus `extra` names."""
    names = ["x", "y", "z"] + (["nx", "ny", "nz"] if normals else []) + ["f_dc_0", "f_dc_1", "f_dc_2"]
    names += [f"f_rest_{i}" for i in range(SH_REST_FLOATS[sh_degree])]
    names += ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    return names + list(extra)


def narrow_table(table62: np.ndarray, sh_degree: int, normals: bool = True) -> np.ndarray:
    """The vertex table of degree `sh_degree` (degree_properties order) that holds the coefficients of a standard 62-property table up to
    that degree: the table a lower-degree PLY of the same splats holds.  Its coefficients above the degree are dropped."""
    t = np.asarray(table62, dtype=np.float32)
    k = SH_REST_FLOATS[sh_degree] // 3
    rest = t[:, 9:54].reshape(-1, 3, 15)[:, :, :k].reshape(t.shape[0], 3 * k)
    cols = [t[:, 0:3]] + ([t[:, 3:6]] if normals else []) + [t[:, 6:9], rest, t[:, 54:62]]
    return np.ascontiguousarray(np.concatenate(cols, axis=1), dtype=np.float32)


def default_properties(nprops: int = 62) -> list[str]:
    names = ["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"] + [f"f_rest_{i}" for i in range(45)]
    names += ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"]
    return names[:nprops]


def _basis_mul(a, b):
    """Godot Basis*Basis, rows[i][j] = b[0][j]*a[i][0] + b[1][j]*a[i][1] + b[2][j]*a[i][2] (float32)."""
    o = [[None] * 3 for _ in range(3)]
    for i in range(3):
        for j in range(3):
            o[i][j] = (b[0][j] * a[i][0] + b[1][j] * a[i][1]) + b[2][j] * a[i][2]
    return o


def swizzle_splats(p: np.ndarray, creation_time: float, layout: PlyLayout | None = None) -> np.ndarray:
    """util/ply_file.gd:41-69 for a block of vertices. p: (m, nprops) float32 -> (m, 60) float32.  layout: PlyFile.layout() of the
    table (default: the standard 62-property layout); SH coefficients above the file's degree are zero.  A layout with filter_3d >= 0
    folds Mip-Splatting's 3D filter into scale and opacity with the float64 operations of gsr_upload_ply_filtered."""
    p = np.asarray(p, dtype=np.float32)
    L = layout or PLY_LAYOUT_3DGS
    m = p.shape[0]
    out = np.zeros((m, STRUCT_SIZE), dtype=np.float32)
    out[:, 0:3] = p[:, L.x:L.x + 3]
    out[:, 3] = F(creation_time)
    # exp() is a GDScript float (float64); narrowed when stored in Vector3 (real_t = float32)
    with np.errstate(over="ignore"):
        e = [np.exp(p[:, L.scale + k].astype(np.float64)) for k in range(3)]
        sigmoid = 1.0 / (1.0 + np.exp(-p[:, L.opacity].astype(np.float64)))
    opacity = sigmoid.astype(np.float32)
    if L.filter_3d >= 0:   # Mip-Splatting: q'_i = exp(scale_i)^2 + f^2 for the splats with f > 0
        f = p[:, L.filter_3d].astype(np.float64)
        on = f > 0.0
        with np.errstate(over="ignore", under="ignore", invalid="ignore"):
            q = [ek * ek for ek in e]
            g = [qk + f * f for qk in q]
            coef = np.sqrt(((q[0] * q[1]) * q[2]) / ((g[0] * g[1]) * g[2]))
            e = [np.where(on, np.sqrt(gk), ek) for gk, ek in zip(g, e)]
            opacity = np.where(on, sigmoid * coef, sigmoid).astype(np.float32)
    sc = [ek.astype(np.float32) for ek in e]
    qx, qy, qz, qw = p[:, L.rot + 1], p[:, L.rot + 2], p[:, L.rot + 3], p[:, L.rot]  # Quaternion(rot_1, rot_2, rot_3, rot_0)
    d = ((qx * qx + qy * qy) + qz * qz) + qw * qw
    s = F(2.0) / d
    xs, ys, zs = qx * s, qy * s, qz * s
    wx, wy, wz = qw * xs, qw * ys, qw * zs
    xx, xy, xz = qx * xs, qx * ys, qx * zs
    yy, yz, zz = qy * ys, qy * zs, qz * zs
    one = F(1.0)
    B = [[one - (yy + zz), xy - wz, xz + wy], [xy + wz, one - (xx + zz), yz - wx], [xz - wy, yz + wx, one - (xx + yy)]]
    R = [[B[c][r] for c in range(3)] for r in range(3)]  # .transposed()
    zero = np.zeros(m, dtype=np.float32)
    S = [[sc[0], zero, zero], [zero, sc[1], zero], [zero, zero, sc[2]]]
    M = _basis_mul(S, R)
    Mt = [[M[c][r] for c in range(3)] for r in range(3)]
    Cv = _basis_mul(Mt, M)
    out[:, 4], out[:, 5], out[:, 6] = Cv[0][0], Cv[0][1], Cv[0][2]
    out[:, 7], out[:, 8], out[:, 9] = Cv[1][1], Cv[1][2], Cv[2][2]
    out[:, 10] = opacity
    out[:, 12:15] = p[:, L.f_dc:L.f_dc + 3]
    k = SH_REST_FLOATS[L.sh_degree] // 3
    if k:
        rest = p[:, L.f_rest:L.f_rest + 3 * k].reshape(m, 3, k)  # channel-major in the file
        out[:, 15:15 + 3 * k] = rest.transpose(0, 2, 1).reshape(m, 3 * k)  # coefficient-major RGB
    return out


def load_gaussian_splats(point_cloud: PlyFile, stride: int, upload, should_terminate=None, num_points_loaded=None,
                         callback=None, clock=None, layout: PlyLayout | None = None) -> None:
    """util/ply_file.gd:28-77.  `upload(first_splat, block60)` plays the role of device.buffer_update
    (:71); `clock()` returns seconds (Time.get_ticks_msec()*1e-3, :40) and stamps each chunk."""
    assert stride >= 1, "stride must be >= 1 (the reference requires size >= 1000)"
    table = point_cloud.table
    n = point_cloud.size
    i = 0
    while i * stride < n:
        if should_terminate is not None and should_terminate[0]:
            return
        lo, hi = i * stride, min(n, (i + 1) * stride)
        block = swizzle_splats(table[lo:hi], clock() if clock else 0.0, layout)
        if should_terminate is not None and should_terminate[0]:
            return
        upload(lo, block)
        if num_points_loaded is not None:
            num_points_loaded[0] += hi - lo
        i += 1
    if callback:
        callback()
