"""SuperSplat / PlayCanvas `compressed.ply` files (include/gsr.h "Compressed PLY").

A `CompressedPlyFile` holds the three element bodies of the file as numpy arrays: `chunks` (float32, one row of 18 or 12 floats per
256 splats), `packed` (uint32, 4 words per splat: position, rotation, scale, colour) and `sh` (uint8, 3((d+1)^2 - 1) bytes per splat, or
None at degree 0).  `GaussianSplattingRasterizer.export_compressed_ply()` makes one on the GPU and `upload_compressed_ply()` loads one;
`save` and `parse` write and read the file.  PlyFile (the float 3DGS PLY) is a separate class.
"""
from __future__ import annotations

import numpy as np

CHUNK = 256
CHUNK_PROPERTIES = ["min_x", "min_y", "min_z", "max_x", "max_y", "max_z",
                    "min_scale_x", "min_scale_y", "min_scale_z", "max_scale_x", "max_scale_y", "max_scale_z",
                    "min_r", "min_g", "min_b", "max_r", "max_g", "max_b"]
VERTEX_PROPERTIES = ["packed_position", "packed_rotation", "packed_scale", "packed_color"]
SH_BYTES = (0, 9, 24, 45)   # per splat, SH degree 0..3


class CompressedPlyFile:
    """Attributes: chunks (C, 18 or 12) float32, packed (size, 4) uint32, sh (size, 3((d+1)^2 - 1)) uint8 or None, sh_degree, size."""

    def __init__(self, path: str = ""):
        self.chunks = np.zeros((0, 18), dtype=np.float32)
        self.packed = np.zeros((0, 4), dtype=np.uint32)
        self.sh = None
        self.sh_degree = 0
        self.size = 0
        if path:
            self.parse(path)

    @classmethod
    def from_arrays(cls, chunks, packed, sh=None, sh_degree: int = 0) -> "CompressedPlyFile":
        self = cls()
        self.packed = np.ascontiguousarray(packed, dtype=np.uint32).reshape(-1, 4)
        self.size = int(self.packed.shape[0])
        c = np.asarray(chunks, dtype=np.float32)
        self.chunks = np.ascontiguousarray(c.reshape(-1, c.shape[-1] if c.ndim == 2 else 18))
        self.sh_degree = int(sh_degree)
        self.sh = None if self.sh_degree == 0 else np.ascontiguousarray(sh, dtype=np.uint8).reshape(self.size, SH_BYTES[self.sh_degree])
        if self.chunks.shape != ((self.size + CHUNK - 1) // CHUNK, self.chunks.shape[1]) or self.chunks.shape[1] not in (12, 18):
            raise ValueError(f"{self.chunks.shape} chunk floats for {self.size} splats")
        return self

    @property
    def chunk_floats(self) -> int:
        return int(self.chunks.shape[1])

    def header(self) -> bytes:
        lines = ["ply", "format binary_little_endian 1.0", f"element chunk {self.chunks.shape[0]}"]
        lines += [f"property float {p}" for p in CHUNK_PROPERTIES[:self.chunk_floats]]
        lines += [f"element vertex {self.size}"] + [f"property uint {p}" for p in VERTEX_PROPERTIES]
        if self.sh_degree > 0:
            lines += [f"element sh {self.size}"] + [f"property uchar f_rest_{i}" for i in range(SH_BYTES[self.sh_degree])]
        return ("\n".join(lines + ["end_header"]) + "\n").encode("ascii")

    def save(self, path: str) -> None:
        with open(path, "wb") as f:
            f.write(self.header())
            f.write(np.ascontiguousarray(self.chunks, dtype="<f4").tobytes())
            f.write(np.ascontiguousarray(self.packed, dtype="<u4").tobytes())
            if self.sh_degree > 0:
                f.write(np.ascontiguousarray(self.sh, dtype=np.uint8).tobytes())

    def parse(self, path: str) -> None:
        elements = []   # [name, count, [properties]]
        with open(path, "rb") as f:
            if f.readline().strip() != b"ply":
                raise ValueError(f"{path} is not a PLY file")
            while True:
                raw = f.readline()
                if not raw:
                    raise ValueError("PLY header has no end_header")
                line = raw.decode("ascii", "replace").strip().split()
                if not line or line[0] == "comment":
                    continue
                if line[0] == "end_header":
                    break
                if line[0] == "format" and line[1] != "binary_little_endian":
                    raise ValueError(f"compressed PLY must be binary_little_endian, not {line[1]}")
                if line[0] == "element":
                    elements.append([line[1], int(line[2]), []])
                elif line[0] == "property":
                    elements[-1][2].append(line[-1])
            body = {}
            for name, count, props in elements:
                dt = {"chunk": "<f4", "vertex": "<u4", "sh": "u1"}.get(name)
                if dt is None:
                    raise ValueError(f"unexpected element {name}")
                a = np.fromfile(f, dtype=dt, count=count * len(props))
                if a.size != count * len(props):
                    raise ValueError(f"compressed PLY body truncated in element {name}")
                body[name] = a.reshape(count, len(props))
        if "chunk" not in body or "vertex" not in body or body["vertex"].shape[1] != 4:
            raise ValueError("compressed PLY needs a chunk element and a vertex element of 4 packed words")
        sh = body.get("sh")
        degree = SH_BYTES.index(sh.shape[1]) if sh is not None else 0
        other = CompressedPlyFile.from_arrays(body["chunk"], body["vertex"], sh, degree)
        self.chunks, self.packed, self.sh, self.sh_degree, self.size = other.chunks, other.packed, other.sh, other.sh_degree, other.size


def is_compressed_ply(path: str) -> bool:
    """Whether the PLY header at `path` declares SuperSplat's chunk element and packed vertex words."""
    try:
        with open(path, "rb") as f:
            head = f.read(4096)
    except OSError:
        return False
    text = head.split(b"end_header")[0]
    return text.startswith(b"ply") and b"element chunk" in text and b"property uint packed_position" in text
