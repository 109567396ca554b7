"""Skeletons of `skeletonize` and `aggregate-skeleton-fragments` (reference plugins/skeletonize.py and
plugins/aggregate_skeleton_fragments.py, which go through kimimaro and cloudvolume; neither is a dependency here).

``Skeleton`` holds vertices (float32 (N, 3) x, y, z in physical units), edges (uint32 (M, 2)) and radii (float32 (N,)).  Its
precomputed form follows the layout of cloudvolume's published ``Skeleton.to_precomputed``: uint32 vertex count, uint32 edge
count, float32 vertices, uint32 edges, float32 radii, uint8 vertex types (all 0).  Those bytes are not pinned against
cloudvolume, which is not installed.
"""
from __future__ import annotations

import math
import os
import re
import struct
from collections import defaultdict

import numpy as np

from .mesh import local_path


def check_params(scale, const, pdrf_scale, pdrf_exponent, dust_threshold, voxel_size=(1, 1, 1), shape=(1, 1, 1)) -> None:
    """The parameter rules of skeletonize (ValueError before any kernel runs), csrc/skeleton.cu's among them: the geodesic field
    stays finite and strictly increasing when (pdrf_scale + 1) * diagonal step * voxels * (1 + 2^-19) < 2^53 * the smallest
    voxel size (DESIGN.md f10)."""
    for name, v in (("scale", scale), ("const", const), ("pdrf_scale", pdrf_scale)):
        if isinstance(v, bool) or not (math.isfinite(float(v)) and float(v) >= 0):
            raise ValueError(f"skeletonize: {name} is a finite number >= 0, not {v}")
    if isinstance(pdrf_exponent, bool) or int(pdrf_exponent) != pdrf_exponent or not 1 <= int(pdrf_exponent) <= 16:
        raise ValueError(f"skeletonize: pdrf_exponent is an integer from 1 to 16, not {pdrf_exponent}")
    if isinstance(dust_threshold, bool) or int(dust_threshold) != dust_threshold or int(dust_threshold) < 0:
        raise ValueError(f"skeletonize: dust_threshold is an integer >= 0, not {dust_threshold}")
    w = tuple(float(v) for v in voxel_size)
    if len(w) != 3 or not all(math.isfinite(v) and v > 0 for v in w):
        raise ValueError(f"skeletonize: the voxel size is three positive finite numbers, not {voxel_size}")
    if not geodesic_is_bounded(float(pdrf_scale), w, math.prod(int(v) for v in shape)):
        raise ValueError("skeletonize: D must stay finite and strictly increasing: (pdrf_scale + 1) * diagonal step * chunk voxels * "
                         "(1 + 2^-19) must be below 2^53 * the smallest voxel size")


def geodesic_is_bounded(pdrf_scale: float, w, voxels: int) -> bool:
    a, b, c = w[0] * w[0], w[1] * w[1], w[2] * w[2]
    diagonal = math.sqrt((a + b) + c)
    bound = (((pdrf_scale + 1.0) * diagonal) * float(voxels)) * (1.0 + 2.0 ** -19)
    return math.isfinite(diagonal) and bound < 2.0 ** 53 * min(w)


class Skeleton:
    def __init__(self, vertices=None, edges=None, radii=None):
        self.vertices = np.ascontiguousarray(np.zeros((0, 3)) if vertices is None else vertices, np.float32).reshape(-1, 3)
        self.edges = np.ascontiguousarray(np.zeros((0, 2)) if edges is None else edges, np.uint32).reshape(-1, 2)
        self.radii = np.ascontiguousarray(np.zeros(len(self.vertices)) if radii is None else radii, np.float32).reshape(-1)
        if len(self.radii) != len(self.vertices):
            raise ValueError("a skeleton has one radius per vertex")
        if self.edges.size and int(self.edges.max()) >= len(self.vertices):
            raise ValueError("an edge names a vertex the skeleton does not have")

    def __eq__(self, other) -> bool:
        return (isinstance(other, Skeleton) and np.array_equal(self.vertices, other.vertices) and np.array_equal(self.edges, other.edges)
                and np.array_equal(self.radii, other.radii))

    def __repr__(self) -> str:
        return f"Skeleton(vertices={len(self.vertices)}, edges={len(self.edges)})"

    def translated(self, offset_xyz) -> "Skeleton":
        return Skeleton(self.vertices + np.asarray(offset_xyz, np.float32), self.edges, self.radii)

    def to_precomputed(self) -> bytes:
        nv, ne = len(self.vertices), len(self.edges)
        return (struct.pack("<II", nv, ne) + self.vertices.astype("<f4").tobytes() + self.edges.astype("<u4").tobytes()
                + self.radii.astype("<f4").tobytes() + np.zeros(nv, np.uint8).tobytes())

    @classmethod
    def from_precomputed(cls, data: bytes) -> "Skeleton":
        nv, ne = struct.unpack_from("<II", data, 0)
        off = 8
        v = np.frombuffer(data, "<f4", 3 * nv, off).reshape(nv, 3)
        off += 12 * nv
        e = np.frombuffer(data, "<u4", 2 * ne, off).reshape(ne, 2)
        off += 8 * ne
        r = np.frombuffer(data, "<f4", nv, off) if len(data) >= off + 4 * nv else np.zeros(nv, np.float32)
        return cls(v, e, r)

    def to_swc(self) -> str:
        """SWC: one line per vertex, ``n type x y z radius parent`` with 1-based n and parent -1 for a tree's root.  An edge
        (v, p) makes p the parent of v (the rows of `skeletonize`); a vertex without one is a root."""
        parent = np.full(len(self.vertices), -1, np.int64)
        for v, p in self.edges.tolist():
            if parent[v] < 0:
                parent[v] = p
        lines = ["# skeleton written by chunkflow_b200"]
        for i, (x, y, z) in enumerate(self.vertices.tolist()):
            par = int(parent[i]) + 1 if parent[i] >= 0 else -1
            lines.append(f"{i + 1} 0 {x!r} {y!r} {z!r} {float(self.radii[i])!r} {par}")
        return "\n".join(lines) + "\n"

    @classmethod
    def merge(cls, fragments) -> "Skeleton":
        """The fragments concatenated, vertices with equal coordinates merged (the first one's radius kept, vertices in order of
        first appearance) and duplicate edges dropped (an edge is unordered; self-loops go)."""
        coords, radii, index, edges = [], [], {}, set()
        for f in fragments:
            local = []
            for p, r in zip(map(tuple, f.vertices.tolist()), f.radii.tolist()):
                if p not in index:
                    index[p] = len(coords)
                    coords.append(p)
                    radii.append(r)
                local.append(index[p])
            for a, b in f.edges.tolist():
                a, b = local[a], local[b]
                if a != b:
                    edges.add((min(a, b), max(a, b)))
        return cls(np.array(coords, np.float32).reshape(-1, 3), np.array(sorted(edges), np.uint32).reshape(-1, 2), np.array(radii, np.float32))


def bbox_string(voxel_offset, shape) -> str:
    """The chunk's bounding box as the reference's ``bbox.string`` (cloudvolume's Bbox.to_filename): ``z0-z1_y0-y1_x0-x1``."""
    return "_".join(f"{int(a)}-{int(a) + int(n)}" for a, n in zip(voxel_offset, shape))


def write_fragments(skeletons: dict, output_path: str, voxel_offset, shape, voxel_size, output_format: str = "precomputed") -> list:
    """``{id}:{bbox}`` fragment files (``.swc`` added for swc) with vertices shifted by voxel offset * voxel size -> the names."""
    if output_format not in ("precomputed", "swc"):
        raise ValueError(f"unsupported skeleton format {output_format}")
    path = local_path(output_path)
    os.makedirs(path, exist_ok=True)
    shift = (np.asarray(voxel_offset, np.float64) * np.asarray(voxel_size, np.float64))[::-1].astype(np.float32)
    names = []
    for i in sorted(skeletons):
        s = skeletons[i].translated(shift)
        name = f"{i}:{bbox_string(voxel_offset, shape)}"
        if output_format == "swc":
            name += ".swc"
            data = s.to_swc().encode()
        else:
            data = s.to_precomputed()
        with open(os.path.join(path, name), "wb") as f:
            f.write(data)
        names.append(name)
    return names


def aggregate_fragments(fragments_path: str, output_path: str, prefix: str = "") -> dict:
    """Every skeleton id's precomputed fragments under ``fragments_path`` (names starting with ``prefix``; the id is the
    reference's ``(\\d+):`` match) merged into ``output_path/{id}``.  kimimaro.postprocess (dust and tick removal, joining) is
    not applied.  -> {id: Skeleton}."""
    src, dst = local_path(fragments_path), local_path(output_path)
    groups = defaultdict(list)
    for name in sorted(os.listdir(src)):
        if not name.startswith(prefix or ""):
            continue
        m = re.search(r"(\d+):", name)
        if m:
            groups[int(m.group(1))].append(name)
    os.makedirs(dst, exist_ok=True)
    out = {}
    for sid in sorted(groups):
        frags = []
        for name in groups[sid]:
            with open(os.path.join(src, name), "rb") as f:
                frags.append(Skeleton.from_precomputed(f.read()))
        out[sid] = Skeleton.merge(frags)
        with open(os.path.join(dst, str(sid)), "wb") as f:
            f.write(out[sid].to_precomputed())
    return out
