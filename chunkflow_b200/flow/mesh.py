"""The files of `mesh` (reference flow/mesh.py, MeshOperator): one chunk's meshes written as neuroglancer's legacy precomputed
fragments, as obj or as ply, on a local path.  The reference writes through CloudFiles and zmesh, neither of which this project
depends on; the formats are restated here (oracle/mesh_oracle.py holds the same rules):

    precomputed  uint32 vertex count, float32 x y z per vertex, uint32 indices, gzip-compressed as ``<name>.gz`` (what
                 CloudFiles does with compress='gzip' on a local path); vertices shifted by voxel offset * voxel size
    obj          ``v x y z`` lines, then ``f i j k`` lines, 1-based
    ply          binary little endian: float x, y, z; faces as a uchar count and uint indices

The exact bytes of zmesh's to_obj / to_ply are not pinned.
"""
from __future__ import annotations

import gzip
import json
import os
import pickle
import struct

import numpy as np


def local_path(path: str) -> str:
    """A local directory or ``file://`` URL -> the directory; any other protocol is refused."""
    if path.startswith("file://"):
        return path[len("file://"):]
    if "://" in path:
        raise ValueError(f"mesh: only local paths and file:// are supported, not {path}")
    return path


def to_precomputed(vertices, faces) -> bytes:
    v = np.ascontiguousarray(vertices, "<f4")
    return struct.pack("<I", v.shape[0]) + v.tobytes() + np.ascontiguousarray(faces, "<u4").tobytes()


def to_obj(vertices, faces) -> bytes:
    lines = ["v {} {} {}".format(*(repr(float(c)) for c in v)) for v in np.asarray(vertices, np.float32)]
    lines += ["f {} {} {}".format(*(int(i) + 1 for i in f)) for f in np.asarray(faces, np.uint32)]
    return ("\n".join(lines) + "\n").encode()


def to_ply(vertices, faces) -> bytes:
    v, f = np.asarray(vertices, "<f4"), np.asarray(faces, "<u4")
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {v.shape[0]}\nproperty float x\nproperty float y\nproperty float z\n"
              f"element face {f.shape[0]}\nproperty list uchar uint vertex_indices\nend_header\n").encode()
    rec = np.zeros(f.shape[0], dtype=[("n", "u1"), ("i", "<u4", 3)])
    rec["n"], rec["i"] = 3, f
    return header + np.ascontiguousarray(v).tobytes() + rec.tobytes()


def bbox_string(start, stop) -> str:
    """cloudvolume's Bbox.to_filename: ``a0-b0_a1-b1_a2-b2``."""
    return "_".join(f"{int(a)}-{int(b)}" for a, b in zip(start, stop))


class MeshWriter:
    """Where and how MeshOperator writes: for precomputed, the ``mesh`` directory named in the ``info`` file at the output path
    (``mesh_err_{e}`` is added to it when missing) and the voxel size of ``scales[mip]`` (x, y, z there)."""

    def __init__(self, output_path: str, output_format: str, mip: int = 0, voxel_size=None, max_simplification_error=40,
                 manifest: bool = False, shard: bool = False):
        if output_format not in ("precomputed", "ply", "obj"):
            raise ValueError(f"unsupported format {output_format}")
        if manifest or shard:
            assert output_format == "precomputed"
        self.output_format, self.manifest, self.shard = output_format, manifest, shard
        path = local_path(output_path)
        self.voxel_size = None if voxel_size is None else tuple(voxel_size)
        self.mesh_path = path
        if output_format == "precomputed":
            with open(os.path.join(path, "info")) as f:
                info = json.load(f)
            if "mesh" not in info:
                info["mesh"] = f"mesh_err_{max_simplification_error}"
                with open(os.path.join(path, "info"), "w") as f:
                    json.dump(info, f)
            self.mesh_path = os.path.join(path, info["mesh"])
            self.voxel_size = tuple(info["scales"][mip]["resolution"])[::-1]   # (z, y, x)
        os.makedirs(self.mesh_path, exist_ok=True)

    def _put(self, name: str, data: bytes, compress: bool = False) -> None:
        with open(os.path.join(self.mesh_path, name + (".gz" if compress else "")), "wb") as f:
            f.write(gzip.compress(data, mtime=0) if compress else data)

    def write(self, meshes: dict, voxel_offset, shape, skip_ids=()) -> None:
        """The files of one chunk's meshes (``{id: (vertices xyz in the chunk's frame, faces)}``)."""
        offset = np.asarray(voxel_offset, np.int64)
        stop = offset + np.asarray(shape, np.int64)
        vs = np.asarray(self.voxel_size, np.float64)

        def data(v, fc):
            if self.output_format == "precomputed":
                v = np.asarray(v, np.float32) + (offset[::-1] * vs[::-1]).astype(np.float32)
                return to_precomputed(v, fc), v
            return (to_ply if self.output_format == "ply" else to_obj)(v, fc), v

        if self.shard:
            frags, boxes = [], {}
            for i in sorted(meshes):
                d, v = data(*meshes[i])
                frags.append(d)
                boxes[str(i)] = [v.min(0).tolist(), v.max(0).tolist()] if len(v) else [[0.0] * 3, [0.0] * 3]
            name = bbox_string(offset, stop)
            with open(os.path.join(self.mesh_path, f"{name}.frags"), "wb") as f:
                f.write(gzip.compress(pickle.dumps(frags), mtime=0))
            with open(os.path.join(self.mesh_path, f"{name}.spatial"), "wb") as f:
                f.write(gzip.compress(json.dumps(boxes).encode(), mtime=0))
            return
        skip = {int(i) for i in (skip_ids or ())}
        for i in sorted(meshes):
            if i in skip:
                continue
            d, _ = data(*meshes[i])
            if self.output_format == "precomputed":
                name = f"{i}:0:{bbox_string(offset[::-1], stop[::-1])}"
                self._put(name, d, compress=True)
            else:
                name = f"{i}.{self.output_format}"
                self._put(name, d)
            if self.manifest:
                self._put(f"{i}:0", json.dumps({"fragments": [name]}).encode())
                self._put("info", json.dumps({"@type": "neuroglancer_legacy_mesh"}).encode())
