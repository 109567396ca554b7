"""`mesh` on the CPU: the case table of csrc/mesh_kernels.cuh against the generator of oracle/mesh_oracle.py and its surface
properties; known answers and invariants of the oracle's marching cubes; csrc/mesh.cu, compiled for the host behind the
one-lane CUDA shim (tests/host_emulation), against the oracle; the native simplifier against the oracle's; the writers."""
import collections
import gzip
import json
import os
import pickle
import re
import struct

import numpy as np
import pytest

import host_emulation
from chunkflow_b200 import _native as N
from oracle import mesh_oracle as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = host_emulation.build("mesh", tmp_path_factory)
    N.bind_mesh(lib)
    return lib


def emu_mesh(lib, seg, voxel_size=(1, 1, 1), skip=(), close=False):
    """The library's own sequence (count, allocate, weld, read) on host buffers."""
    seg = np.ascontiguousarray(seg)
    if seg.dtype.kind == "i":
        seg = seg.view(seg.dtype.str.replace("i", "u"))
    code = N.DTYPE_U64 if seg.dtype.itemsize == 8 else N.DTYPE_U32
    sk = np.array(sorted({int(i) % 2 ** 64 for i in skip}), np.uint64)
    work = np.zeros(N.mesh_workspace(seg.shape, close, lib), np.uint8)
    args = (seg.ctypes.data, code, seg.shape, sk.ctypes.data if sk.size else 0, sk.size, close)
    counts = N.mesh_count_device(*args, work.ctypes.data, lib=lib)
    nbytes = N.mesh_buffer_bytes(counts, lib=lib)
    buf = np.zeros(nbytes, np.uint8)
    n = N.mesh_device(*args, voxel_size, work.ctypes.data, counts, buf.ctypes.data, nbytes, lib=lib)
    return N.mesh_read(buf.ctypes.data, counts, n, lib=lib)


def assert_same(a: dict, b: dict):
    assert list(a) == list(b)
    for k in a:
        assert a[k][0].dtype == np.float32 and a[k][1].dtype == np.uint32
        assert np.array_equal(a[k][0], b[k][0]), k
        assert np.array_equal(a[k][1], b[k][1]), k


def edge_counts(faces):
    return collections.Counter(map(tuple, M.directed_edges(faces).tolist()))


def is_closed_oriented(faces) -> bool:
    cnt = edge_counts(faces)
    return all(n == 1 and cnt.get((b, a)) == 1 for (a, b), n in cnt.items())


def blobs(shape, seed, n=6):
    rng = np.random.default_rng(seed)
    z, y, x = np.indices(shape)
    seg = np.zeros(shape, np.uint32)
    for i in range(1, n + 1):
        c, r = rng.uniform(0, shape), rng.uniform(1.5, max(2.0, max(shape) / 2.5), 3)
        seg[((z - c[0]) / r[0]) ** 2 + ((y - c[1]) / r[1]) ** 2 + ((x - c[2]) / r[2]) ** 2 < 1] = i
    return seg


# ------------------------------------------------------------------------------------------------------------
# the table
# ------------------------------------------------------------------------------------------------------------
def embedded_table():
    with open(os.path.join(ROOT, "chunkflow_b200", "csrc", "mesh_kernels.cuh")) as f:
        text = f.read()
    body = text[text.index("#define CFB_MC_TABLE"):text.index("McCase kMcTable[256] = CFB_MC_TABLE")]
    nums = [int(v) for v in re.findall(r"\d+", body.split("{", 1)[1])]
    arr = np.array(nums).reshape(256, 1 + 3 * M.MAX_TRIANGLES)
    return arr[:, 0].astype(np.uint8), arr[:, 1:].reshape(256, M.MAX_TRIANGLES, 3).astype(np.uint8)


def test_embedded_table_equals_the_generated_one():
    counts, edges = embedded_table()
    g_counts, g_edges = M.build_table()
    assert np.array_equal(counts, g_counts)
    assert np.array_equal(edges, g_edges)
    assert counts[0] == 0 and counts[255] == 0 and counts[1] == 1


def test_every_case_is_an_oriented_patch_bounded_by_the_cube_faces():
    faces = M._faces()
    for m in range(256):
        tris = M.case_triangles(m)
        cnt = edge_counts(np.array(tris, np.int64).reshape(-1, 3))
        assert all(n == 1 for n in cnt.values()), m                      # oriented: no directed edge twice
        border = [(a, b) for (a, b) in cnt if (b, a) not in cnt]
        segs = {(b, a) for f in range(6) for a, b in M.face_segments(m, f)}
        assert set(border) == segs, m                 # the boundary is the face segments (walked the other way round)
        for a, b in border:
            assert any(a in es and b in es for _, es in faces), m        # ... which lie on a cube face
        cut = {e for e, (c0, c1, _) in enumerate(M.EDGES) if ((m >> c0) & 1) != ((m >> c1) & 1)}
        assert {e for t in tris for e in t} == cut, m                     # every cut edge carries a vertex


def test_face_segments_depend_on_the_face_corners_only():
    for f, (n, es) in enumerate(M._faces()):
        corners = sorted({c for e in es for c in M.EDGES[e][:2]})
        seen = {}
        for m in range(256):
            key = tuple((m >> c) & 1 for c in corners)
            segs = sorted(M.face_segments(m, f))
            assert seen.setdefault(key, segs) == segs


# ------------------------------------------------------------------------------------------------------------
# known answers and invariants of the oracle
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name, seg, verts, faces, volume", [
    ("voxel", np.ones((1, 1, 1)), 6, 8, 1 / 6),
    ("bar", np.ones((1, 1, 2)), 10, 16, 2 / 3),
    ("L", np.array([[[1, 1], [1, 0]]]), 14, 24, 1.25),
    ("block", np.ones((2, 2, 2)), 24, 44, 17 / 3),
    ("diagonal", np.array([[[1, 0], [0, 0]], [[0, 0], [0, 1]]]), 12, 16, 1 / 3),
])
def test_known_answers(name, seg, verts, faces, volume):
    v, f = M.marching_cubes(seg.astype(np.uint32), (2, 3, 5), close=True)[1]
    assert (len(v), len(f)) == (verts, faces)
    assert M.signed_volume(v, f) == pytest.approx(volume * 30, rel=1e-12)
    assert is_closed_oriented(f)


def test_single_voxel_is_an_octahedron_at_the_voxel_faces():
    v, f = M.marching_cubes(np.ones((1, 1, 1), np.uint32), (2, 3, 5), close=True)[1]
    assert sorted(map(tuple, v.tolist())) == sorted([(2.5, 1.5, 0.0), (2.5, 0.0, 1.0), (0.0, 1.5, 1.0), (5.0, 1.5, 1.0),
                                                     (2.5, 3.0, 1.0), (2.5, 1.5, 2.0)])
    assert M.signed_volume(v, f) == 2 * 3 * 5 / 6


def test_zero_and_skipped_ids_give_nothing():
    seg = np.zeros((3, 4, 5), np.uint64)
    assert M.marching_cubes(seg, close=True) == {}
    seg[1, 1:3, 1:4] = 7
    seg[0, 0, 0] = 2 ** 64 - 1
    assert list(M.marching_cubes(seg, close=True)) == [7, 2 ** 64 - 1]
    assert list(M.marching_cubes(seg, skip_ids=[7, -1], close=True)) == []


@pytest.mark.parametrize("kind", ["random", "blobs", "salt"])
@pytest.mark.parametrize("wide", [False, True])
def test_closed_meshes_are_oriented_manifolds_with_positive_volume(kind, wide):
    rng = np.random.default_rng(3)
    shape = (7, 9, 11)
    if kind == "random":
        seg = rng.integers(0, 4, shape).astype(np.uint32)
    elif kind == "blobs":
        seg = blobs(shape, 5)
    else:
        seg = np.where(rng.random(shape) < 0.1, rng.integers(1, 1000, shape), 0).astype(np.uint32)
    if wide:
        seg = np.where(seg > 0, np.uint64(2 ** 64 - 1) - seg.astype(np.uint64), np.uint64(0))
    meshes = M.marching_cubes(seg, (4, 3, 2), close=True)
    assert len(meshes) == len(np.unique(seg[seg > 0]))
    for k, (v, f) in meshes.items():
        assert is_closed_oriented(f), k
        assert M.signed_volume(v, f) > 0, k


def test_open_meshes_have_borders_only_on_the_outer_planes():
    seg = blobs((8, 10, 12), 7)
    vs = np.array([4.0, 3.0, 2.0])
    lo, hi = 0.5 * vs[::-1], (np.array(seg.shape)[::-1] - 0.5) * vs[::-1]
    for k, (v, f) in M.marching_cubes(seg, vs, close=False).items():
        cnt = edge_counts(f)
        for a, b in [(a, b) for (a, b) in cnt if (b, a) not in cnt]:
            pa, pb = v[a], v[b]
            assert any((pa[i] == pb[i]) and (pa[i] in (lo[i], hi[i])) for i in range(3)), k


# ------------------------------------------------------------------------------------------------------------
# csrc/mesh.cu on the host against the oracle
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 5, 6), (2, 1, 7), (2, 2, 2), (5, 6, 7), (9, 17, 33), (3, 40, 50)])
@pytest.mark.parametrize("close", [False, True])
def test_emulation_equals_the_oracle(emu, shape, close):
    rng = np.random.default_rng(sum(shape))
    for seg in (rng.integers(0, 4, shape).astype(np.uint32), blobs(shape, 1)):
        assert_same(emu_mesh(emu, seg, (40, 4.5, 5), close=close), M.marching_cubes(seg, (40, 4.5, 5), close=close))


def test_emulation_wide_ids_and_skip_ids(emu):
    rng = np.random.default_rng(9)
    seg = rng.integers(0, 5, (6, 13, 11)).astype(np.uint64) + np.uint64(2 ** 64 - 5)
    seg[seg == np.uint64(2 ** 64 - 5)] = 0
    for close in (False, True):
        assert_same(emu_mesh(emu, seg, (1, 2, 3), skip=[-2], close=close), M.marching_cubes(seg, (1, 2, 3), skip_ids=[-2], close=close))
    signed = rng.integers(-3, 3, (5, 6, 7)).astype(np.int32)
    assert_same(emu_mesh(emu, signed, close=True), M.marching_cubes(signed, close=True))


def test_emulation_refuses_bad_arguments(emu):
    seg = np.zeros((2, 2, 2), np.uint32)
    work = np.zeros(N.mesh_workspace(seg.shape, True, emu), np.uint8)
    with pytest.raises(TypeError):
        N.mesh_count_device(seg.ctypes.data, N.DTYPE_F32, seg.shape, 0, 0, False, work.ctypes.data, lib=emu)
    with pytest.raises(N.NativeError):
        N.mesh_count_device(seg.ctypes.data, N.DTYPE_U32, (0, 2, 2), 0, 0, False, work.ctypes.data, lib=emu)
    for zyx in ((2 ** 31, 1, 1), (0, 1, 1)):   # refused through the error code, not an exception across the C ABI
        with pytest.raises(N.NativeError):
            N.mesh_workspace(zyx, False, emu)
    seg[0, 0, 0] = 3
    counts = N.mesh_count_device(seg.ctypes.data, N.DTYPE_U32, seg.shape, 0, 0, True, work.ctypes.data, lib=emu)
    buf = np.zeros(N.mesh_buffer_bytes(counts, lib=emu), np.uint8)
    with pytest.raises(N.NativeError, match="smaller"):
        N.mesh_device(seg.ctypes.data, N.DTYPE_U32, seg.shape, 0, 0, True, (1, 1, 1), work.ctypes.data, counts, buf.ctypes.data,
                      buf.size - 1, lib=emu)
    with pytest.raises(N.NativeError, match="counts"):   # counts that do not match the volume's: no buffer is overrun
        N.mesh_device(seg.ctypes.data, N.DTYPE_U32, seg.shape, 0, 0, True, (1, 1, 1), work.ctypes.data,
                      (counts[0], counts[1] - 1, counts[2]), buf.ctypes.data, buf.size, lib=emu)


# ------------------------------------------------------------------------------------------------------------
# the simplifier
# ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    return N.load()   # the host entry points need no device


def simplify_cases():
    z, y, x = np.indices((14, 16, 18))
    ball = (((z - 7) ** 2 / 30 + (y - 8) ** 2 / 40 + (x - 9) ** 2 / 50) < 1).astype(np.uint32)
    cut = np.zeros((10, 16, 18), np.uint32)
    cut[:, 3:13, 2:16] = ball[:10, 3:13, 2:16] | (z[:10, 3:13, 2:16] < 4)   # touches the chunk's lower z face: an open border
    yield "ball", M.marching_cubes(ball, (40, 4, 4), close=True)[1]
    yield "open", M.marching_cubes(cut, (40, 4, 4), close=False)[1]
    yield "blobs", max(M.marching_cubes(blobs((16, 32, 32), 4, 2), (8, 4, 4), close=False).values(), key=lambda m: len(m[1]))


@pytest.mark.parametrize("factor, error", [(1, 40), (2, 40), (10, 40), (100, 40), (100, 1000), (10, 0.5), (1000, 0)])
def test_native_simplifier_equals_the_oracle(lib, factor, error):
    for name, (v, f) in simplify_cases():
        assert len(f) > 500
        *want, cheapest = M.simplify(v, f, factor, error, next_cost=True)
        got = N.mesh_simplify_host(v, f, factor, error)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), name
        gv, gf = got
        target = -(-len(f) // factor) if factor > 1 else len(f)
        cnt = edge_counts(f)
        border = {a for (a, b) in cnt if (b, a) not in cnt} | {b for (a, b) in cnt if (b, a) not in cnt}
        border_pos = {tuple(v[i]) for i in border}
        if not border:
            assert is_closed_oriented(gf), name
        else:
            assert border_pos <= {tuple(p) for p in gv}, name            # no boundary vertex has moved
            assert all(n == 1 for n in edge_counts(gf).values()), name  # still oriented
        # stopped at the target, or no allowed collapse costs e^2 or less
        assert len(gf) <= target or factor <= 1 or cheapest > float(error) ** 2, name


def test_simplifier_unchanged_below_a_factor_of_two(lib):
    _, (v, f) = next(simplify_cases())
    for factor in (0, 1):
        gv, gf = N.mesh_simplify_host(v, f, factor, 40)
        assert np.array_equal(gv, v) and np.array_equal(gf, f)
    with pytest.raises(TypeError):
        N.mesh_simplify_host(v, f, 2.5, 40)
    with pytest.raises(N.NativeError):
        N.mesh_simplify_host(v[:3], f, 2, 40)   # indices out of range


# ------------------------------------------------------------------------------------------------------------
# the writers
# ------------------------------------------------------------------------------------------------------------
def parse_obj(data: bytes):
    v, f = [], []
    for line in data.decode().splitlines():
        k, *rest = line.split()
        (v if k == "v" else f).append([float(r) for r in rest] if k == "v" else [int(r) - 1 for r in rest])
    return np.array(v, np.float32).reshape(-1, 3), np.array(f, np.uint32).reshape(-1, 3)


def parse_ply(data: bytes):
    head, body = data.split(b"end_header\n", 1)
    nv = int(re.search(rb"element vertex (\d+)", head).group(1))
    nf = int(re.search(rb"element face (\d+)", head).group(1))
    v = np.frombuffer(body[:12 * nv], "<f4").reshape(nv, 3)
    rec = np.frombuffer(body[12 * nv:], dtype=[("n", "u1"), ("i", "<u4", 3)], count=nf)
    assert (rec["n"] == 3).all()
    return v, rec["i"].astype(np.uint32)


def parse_precomputed(data: bytes):
    n = struct.unpack("<I", data[:4])[0]
    v = np.frombuffer(data[4:4 + 12 * n], "<f4").reshape(n, 3)
    return v, np.frombuffer(data[4 + 12 * n:], "<u4").reshape(-1, 3)


def tree(path):
    out = {}
    for d, _, files in os.walk(path):
        for name in files:
            with open(os.path.join(d, name), "rb") as f:
                out[os.path.relpath(os.path.join(d, name), path)] = f.read()
    return out


def make_info(path, resolution=(5, 6, 40)):
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "info"), "w") as f:
        json.dump({"scales": [{"resolution": list(resolution)}, {"resolution": [10, 12, 40]}]}, f)


@pytest.mark.parametrize("fmt, manifest, shard", [("obj", False, False), ("ply", False, False), ("precomputed", False, False),
                                                  ("precomputed", True, False), ("precomputed", False, True)])
def test_writers_round_trip_and_match_the_oracle(tmp_path, fmt, manifest, shard):
    from chunkflow_b200.flow.mesh import MeshWriter
    seg = blobs((6, 10, 12), 2, 3)
    meshes = M.marching_cubes(seg, (40, 6, 5), close=False)
    offset = (3, 20, 10)
    mine, theirs = tmp_path / "mine", tmp_path / "theirs"
    for p in (mine, theirs):
        make_info(str(p)) if fmt == "precomputed" else os.makedirs(p)
    MeshWriter(f"file://{mine}", fmt, voxel_size=(40, 6, 5), max_simplification_error=40, manifest=manifest,
               shard=shard).write(meshes, offset, seg.shape, skip_ids={2})
    M.write(meshes, str(theirs), fmt, offset, seg.shape, (40, 6, 5), manifest=manifest, shard=shard, skip_ids={2})
    a, b = tree(str(mine)), tree(str(theirs))
    assert a == b
    if fmt == "precomputed":
        assert json.loads(a["info"])["mesh"] == "mesh_err_40"
    shift = (np.array(offset)[::-1] * np.array([5, 6, 40])).astype(np.float32)
    if shard:
        frags = pickle.loads(gzip.decompress(a["mesh_err_40/3-9_20-30_10-22.frags"]))
        assert len(frags) == len(meshes)
        spatial = json.loads(gzip.decompress(a["mesh_err_40/3-9_20-30_10-22.spatial"]))
        assert sorted(spatial) == sorted(str(k) for k in meshes)
        return
    for k, (v, f) in meshes.items():
        if k == 2:
            continue
        if fmt == "obj":
            gv, gf = parse_obj(a[f"{k}.obj"])
        elif fmt == "ply":
            gv, gf = parse_ply(a[f"{k}.ply"])
        else:
            name = f"{k}:0:10-22_20-30_3-9"
            gv, gf = parse_precomputed(gzip.decompress(a[f"mesh_err_40/{name}.gz"]))
            v = v + shift
            if manifest:
                assert json.loads(a[f"mesh_err_40/{k}:0"]) == {"fragments": [name]}
                assert json.loads(a["mesh_err_40/info"]) == {"@type": "neuroglancer_legacy_mesh"}
        assert np.array_equal(gv, v) and np.array_equal(gf, f)
    assert not any(n.startswith("2") for n in a)


def test_precomputed_takes_the_resolution_of_the_mip_and_keeps_a_mesh_key(tmp_path):
    from chunkflow_b200.flow.mesh import MeshWriter
    make_info(str(tmp_path))
    with open(tmp_path / "info") as f:
        info = json.load(f)
    info["mesh"] = "meshes"
    with open(tmp_path / "info", "w") as f:
        json.dump(info, f)
    w = MeshWriter(str(tmp_path), "precomputed", mip=1)
    assert w.voxel_size == (40, 12, 10) and w.mesh_path == os.path.join(str(tmp_path), "meshes")


def test_other_protocols_are_refused(tmp_path):
    from chunkflow_b200.flow.mesh import MeshWriter
    with pytest.raises(ValueError, match="only local paths"):
        MeshWriter("gs://bucket/mesh", "obj")


def test_cli_has_the_reference_options():
    from chunkflow_b200.flow.cli import main
    cmd = main.commands["mesh"]
    opts = {o.name: o for o in cmd.params}
    assert opts["output_path"].default == "file:///tmp/mesh/" and opts["output_format"].default == "precomputed"
    assert opts["simplification_factor"].default == 100 and opts["max_simplification_error"].default == 40
    flags = {f for o in cmd.params for f in getattr(o, "opts", [])}
    assert {"--name", "-i", "-m", "--mip", "-v", "--voxel-size", "-o", "-t", "-f", "-e", "-s", "--manifest", "--shard"} <= flags
