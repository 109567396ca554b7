"""`skeletonize` on the CPU: the oracle's distance transform against live scipy, its geodesic field against
scipy.sparse.csgraph.dijkstra, the skeleton properties (a forest with one root per component, every voxel covered by a vertex's
ball); csrc/skeleton.cu, compiled for the host behind the one-lane CUDA shim (tests/host_emulation), against the oracle on
seeded volumes; the writers and the fragment merge."""
import os

import numpy as np
import pytest
from scipy import ndimage
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import dijkstra

import host_emulation
from chunkflow_b200 import _native as N
from chunkflow_b200.flow.skeleton import Skeleton, aggregate_fragments, bbox_string, check_params, write_fragments
from oracle import skeleton_oracle as S


def scipy_dbf(seg, w):
    seg = np.asarray(seg)
    out = np.zeros(seg.shape, np.float32)
    for L in np.unique(seg):
        if L == 0:
            continue
        m = np.pad(seg == L, 1)
        d = ndimage.distance_transform_edt(m, sampling=w)[1:-1, 1:-1, 1:-1].astype(np.float32)
        out[seg == L] = d[seg == L]
    return out


def blobs(shape, seed, n=5, dtype=np.uint32):
    rng = np.random.default_rng(seed)
    z, y, x = np.indices(shape)
    seg = np.zeros(shape, dtype)
    for i in range(1, n + 1):
        c, r = rng.uniform(0, shape), rng.uniform(1.5, max(2.0, max(shape) / 3), 3)
        seg[((z - c[0]) / r[0]) ** 2 + ((y - c[1]) / r[1]) ** 2 + ((x - c[2]) / r[2]) ** 2 < 1] = i * 7919
    return seg


def tubes(shape, seed, n=3, radius=2.0):
    """Branching tubes: a trunk along x with side branches along y and z, one id per tree."""
    rng = np.random.default_rng(seed)
    z, y, x = np.indices(shape)
    seg = np.zeros(shape, np.uint32)
    for t in range(1, n + 1):
        cz, cy = rng.uniform(radius, shape[0] - radius), rng.uniform(radius, shape[1] - radius)
        seg[(z - cz) ** 2 + (y - cy) ** 2 <= radius ** 2] = t
        for _ in range(2):
            bx = rng.uniform(0, shape[2])
            seg[((z - cz) ** 2 + (x - bx) ** 2 <= radius ** 2) & (y > cy)] = t
    return seg


VOLUMES = {
    "blobs": lambda: blobs((12, 20, 22), 1),
    "blobs_touching_faces": lambda: blobs((9, 14, 16), 2, 8),
    "tubes": lambda: tubes((10, 24, 30), 3),
    "tubes_thin": lambda: tubes((7, 20, 25), 4, 2, 1.2),
    "random_labels": lambda: np.random.default_rng(5).integers(0, 3, (6, 7, 8)).astype(np.uint32),
    "single_voxels": lambda: (np.arange(5 * 6 * 7).reshape(5, 6, 7) % 11 == 0).astype(np.uint32) * np.arange(5 * 6 * 7).reshape(5, 6, 7).astype(np.uint32),
    "all_zero": lambda: np.zeros((4, 5, 6), np.uint32),
    "one_slice": lambda: blobs((1, 20, 21), 6),
    "two_slices": lambda: blobs((2, 17, 15), 7),
    "one_row": lambda: (np.arange(40) // 7 % 3).astype(np.uint32).reshape(1, 1, 40),
    "full": lambda: np.full((5, 6, 7), 3, np.uint32),
    "wide_ids": lambda: (blobs((8, 16, 16), 8).astype(np.uint64) * np.uint64(2 ** 40 + 1)) | np.uint64(2 ** 63),
}

PARAMS = [
    dict(voxel_size=(1, 1, 1), const=2, dust_threshold=0),
    dict(voxel_size=(40, 4, 4), const=20, scale=1, dust_threshold=5),
    dict(voxel_size=(1, 1, 1), const=0, scale=1, pdrf_exponent=1, dust_threshold=3),
    dict(voxel_size=(2.5, 1.25, 0.75), const=1.5, scale=2, pdrf_exponent=7, pdrf_scale=1000, dust_threshold=0),
]


@pytest.mark.parametrize("w", [(1, 1, 1), (40, 4, 4)])
@pytest.mark.parametrize("name", ["blobs_touching_faces", "random_labels", "one_slice", "two_slices", "one_row", "full", "single_voxels"])
def test_oracle_dbf_is_scipy_bit_for_bit(name, w):
    seg = VOLUMES[name]()
    assert np.array_equal(S.distance_transform(seg, w), scipy_dbf(seg, w))


def test_axes_of_length_one_and_two():
    rng = np.random.default_rng(9)
    for shape in [(1, 1, 1), (2, 1, 1), (1, 2, 5), (2, 2, 2), (1, 9, 2), (2, 7, 1)]:
        seg = rng.integers(0, 3, shape).astype(np.uint32)
        for w in [(1, 1, 1), (40, 4, 4)]:
            assert np.array_equal(S.distance_transform(seg, w), scipy_dbf(seg, w)), (shape, w)


@pytest.mark.parametrize("w", [(1, 1, 1), (40, 4, 4), (1.5, 0.75, 2.25)])
def test_oracle_geodesic_field_is_csgraph_dijkstra(w):
    seg = tubes((8, 18, 20), 11)
    ids = S.as_ids(seg)
    dbf = S.distance_transform(ids, w).ravel()
    for L, idx in S.objects(ids, (), 0):
        root, D, parent, P = S.geodesic(idx, dbf, ids.shape, w, 100000.0, 4)
        pos = {int(i): k for k, i in enumerate(idx)}
        rows, cols, vals = [], [], []
        for u in idx.tolist():
            for k, v in S.neighbours(u, ids.shape):
                if v in pos:
                    rows.append(pos[u])
                    cols.append(pos[v])
                    vals.append(S.step_length(S.OFFSETS[k], w) * P[v])
        g = csr_matrix((vals, (rows, cols)), shape=(len(idx), len(idx)))
        ref = dijkstra(g, indices=pos[root])
        assert np.array_equal(ref, np.array([D[i] for i in idx.tolist()]))
        members = set(idx.tolist())
        for v, p in parent.items():   # the parent attains the minimum, and no neighbour of a smaller index does
            if v == root:
                continue
            cost = {u: D[u] + S.step_length(np.subtract(np.unravel_index(v, ids.shape), np.unravel_index(u, ids.shape)), w) * P[v]
                    for _, u in S.neighbours(v, ids.shape) if u in members}
            assert cost[p] == D[v] == min(cost.values())
            assert all(cost[u] > D[v] for u in cost if u < p)
            assert D[p] < D[v]


@pytest.mark.parametrize("name", ["blobs", "tubes", "tubes_thin", "wide_ids"])
@pytest.mark.parametrize("p", PARAMS[:2])
def test_skeletons_are_forests_covering_their_objects(name, p):
    seg = VOLUMES[name]()
    p = dict(p)
    w = p.pop("voxel_size")
    out = S.skeletonize(seg, w, **p)
    ids = S.as_ids(seg)
    dbf = S.distance_transform(ids, w)
    comps = {}
    for L, idx in S.objects(ids, (), p["dust_threshold"]):
        comps.setdefault(L, []).append(idx)
    assert sorted(out) == sorted(comps)
    scale, const = p.get("scale", 4), p.get("const", 500)
    for L, (v, e, r) in out.items():
        assert len(e) == len(v) - len(comps[L])   # a forest: one tree per component
        parent = np.full(len(v), -1)
        for a, b in e.tolist():
            assert a != b and parent[a] < 0
            parent[a] = b
        for a in range(len(v)):   # every vertex reaches a root
            seen = 0
            while parent[a] >= 0:
                a, seen = parent[a], seen + 1
                assert seen <= len(v)
        vox = np.stack(np.unravel_index(np.concatenate(comps[L]), ids.shape), 1).astype(np.float64) * w
        centres = (v.astype(np.float64)[:, ::-1] - 0.5 * np.asarray(w))
        rad = scale * r.astype(np.float64) + const
        d = np.sqrt(((vox[:, None, :] - centres[None]) ** 2).sum(-1))
        assert (d <= rad[None] * (1 + 1e-9)).any(1).all()
        assert np.array_equal(r, dbf.ravel()[np.ravel_multi_index(tuple(np.round(centres / w).astype(int).T), ids.shape)])


# ---- the host emulation of csrc/skeleton.cu against the oracle ----
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    lib = host_emulation.build("skeleton", tmp_path_factory)
    N.bind_skeleton(lib)
    return lib


def emu_skeletonize(lib, seg, voxel_size=(1, 1, 1), skip_ids=(), dust_threshold=1000, stats=None, **kw):
    """The library's own sequence (count, allocate, skeletonize, read) on host buffers."""
    seg = np.ascontiguousarray(seg)
    if seg.dtype.kind == "i":
        seg = seg.view(seg.dtype.str.replace("i", "u"))
    code = N.DTYPE_U64 if seg.dtype.itemsize == 8 else N.DTYPE_U32
    sk = np.array(sorted({int(i) % 2 ** 64 for i in skip_ids}), np.uint64)
    work = np.zeros(N.skeleton_workspace(seg.shape, lib), np.uint8)
    args = (seg.ctypes.data, code, seg.shape, voxel_size)
    counts = N.skeleton_count_device(*args, sk.ctypes.data if sk.size else 0, sk.size, dust_threshold, work.ctypes.data, lib=lib)
    buf = np.zeros(max(counts[2], 1), np.uint8)
    p = {k: kw.get(k, S.DEFAULTS[k]) for k in ("scale", "const", "pdrf_scale", "pdrf_exponent")}
    n, st = N.skeleton_device(*args, p["scale"], p["const"], p["pdrf_scale"], p["pdrf_exponent"], work.ctypes.data, counts, buf.ctypes.data,
                              lib=lib)
    if stats is not None:
        stats.update(st)
    return N.skeleton_read(buf.ctypes.data, seg.shape, voxel_size, counts, n, lib=lib)


def assert_same(got: dict, want: dict):
    assert list(got) == list(want)
    for k in want:
        for a, b in zip(got[k], want[k]):
            assert a.dtype == b.dtype and np.array_equal(a, b), k


def emu_edt(lib, seg, w):
    ids = S.as_ids(seg)
    work = np.zeros(N.edt_workspace(ids.shape, lib), np.uint8)
    out = np.zeros(ids.shape, np.float32)
    N.edt_device(ids.ctypes.data, N.DTYPE_U64, ids.shape, w, out.ctypes.data, work.ctypes.data, lib=lib)
    return out


@pytest.mark.parametrize("name", sorted(VOLUMES))
def test_emulated_distance_transform_equals_the_oracle(emu, name):
    seg = VOLUMES[name]()
    for w in [(1, 1, 1), (40, 4, 4), (1.5, 0.75, 2.25)]:
        assert np.array_equal(emu_edt(emu, seg, w), S.distance_transform(seg, w)), w


@pytest.mark.parametrize("name", sorted(VOLUMES))
def test_emulation_equals_the_oracle(emu, name):
    seg = VOLUMES[name]()
    for p in PARAMS:
        p = dict(p)
        w = p.pop("voxel_size")
        assert_same(emu_skeletonize(emu, seg, w, **p), S.skeletonize(seg, w, **p))


def test_emulation_dust_skip_ids_and_signed_ids(emu):
    seg = blobs((10, 18, 18), 12, 6).astype(np.int64)
    seg[seg > 0] -= 3 * 7919   # negative ids: read by their unsigned bit pattern
    skip = [int(seg.flat[np.flatnonzero(seg)[0]])]
    for dust in (0, 30, 10 ** 9):
        got = emu_skeletonize(emu, seg, (2, 1, 1), skip_ids=skip, dust_threshold=dust, const=3)
        assert_same(got, S.skeletonize(seg, (2, 1, 1), skip_ids=skip, dust_threshold=dust, const=3))
        assert (skip[0] % 2 ** 64) not in got
    assert emu_skeletonize(emu, seg.astype(np.int32), (2, 1, 1), dust_threshold=0, const=3).keys() == \
        S.skeletonize(seg.astype(np.int32), (2, 1, 1), dust_threshold=0, const=3).keys()


def test_emulation_reports_sweeps_rounds_and_paths(emu):
    st = {}
    seg = tubes((10, 30, 40), 13, 2, 1.5)
    got = emu_skeletonize(emu, seg, (1, 1, 1), dust_threshold=0, const=1, scale=1, stats=st)
    assert st["sweeps"] >= 2 and st["rounds"] >= 2 and st["paths"] >= st["rounds"]
    assert st["skeleton_voxels"] == sum(len(v[0]) for v in got.values())


def test_emulation_refuses_bad_arguments(emu):
    seg = np.ones((3, 4, 5), np.uint32)
    work = np.zeros(N.skeleton_workspace(seg.shape, emu), np.uint8)
    for bad in [(0, 1, 1), (-1, -1, -1), (np.nan, 1, 1)]:
        with pytest.raises(N.NativeError, match="voxel size"):
            N.skeleton_count_device(seg.ctypes.data, N.DTYPE_U32, seg.shape, bad, 0, 0, 0, work.ctypes.data, lib=emu)
    with pytest.raises(N.NativeError, match="uint32 or uint64"):
        N.skeleton_count_device(seg.ctypes.data, N.DTYPE_F32, seg.shape, (1, 1, 1), 0, 0, 0, work.ctypes.data, lib=emu)
    with pytest.raises(N.NativeError, match="2\\^32"):
        N.skeleton_workspace((2 ** 16, 2 ** 16, 1), emu)
    counts = N.skeleton_count_device(seg.ctypes.data, N.DTYPE_U32, seg.shape, (1, 1, 1), 0, 0, 0, work.ctypes.data, lib=emu)
    buf = np.zeros(counts[2], np.uint8)
    with pytest.raises(N.NativeError, match="pdrf_exponent"):
        N.skeleton_device(seg.ctypes.data, N.DTYPE_U32, seg.shape, (1, 1, 1), 4, 500, 1e5, 17, work.ctypes.data, counts, buf.ctypes.data, lib=emu)
    with pytest.raises(N.NativeError, match="counts"):
        N.skeleton_device(seg.ctypes.data, N.DTYPE_U32, seg.shape, (1, 1, 1), 4, 500, 1e5, 4, work.ctypes.data, (counts[0] + 1, counts[1], counts[2]),
                          buf.ctypes.data, lib=emu)


def test_parameter_and_size_refusals():
    for bad in [dict(scale=-1), dict(const=float("inf")), dict(pdrf_exponent=0), dict(pdrf_exponent=17), dict(pdrf_exponent=2.5),
                dict(dust_threshold=-1)]:
        p = dict(scale=4, const=500, pdrf_scale=1e5, pdrf_exponent=4, dust_threshold=10)
        p.update(bad)
        with pytest.raises(ValueError):
            check_params(**p)
        with pytest.raises(ValueError):
            S.check_params(**p)
    with pytest.raises(TypeError):
        S.as_ids(np.zeros((2, 2, 2), np.float32))
    with pytest.raises(ValueError):
        S.as_ids(np.zeros((2, 2), np.uint32))


# ---- writers and the fragment merge ----
def test_precomputed_and_swc_round_trip():
    seg = tubes((8, 16, 20), 14)
    sk = {k: Skeleton(*v) for k, v in S.skeletonize(seg, (40, 4, 4), const=10, dust_threshold=0).items()}
    for s in sk.values():
        data = s.to_precomputed()
        nv, ne = len(s.vertices), len(s.edges)
        assert len(data) == 8 + 12 * nv + 8 * ne + 4 * nv + nv
        assert Skeleton.from_precomputed(data) == s
        lines = [ln.split() for ln in s.to_swc().splitlines() if not ln.startswith("#")]
        assert len(lines) == nv and sum(ln[-1] == "-1" for ln in lines) == nv - ne
        assert np.array_equal(np.array([[float(c) for c in ln[2:5]] for ln in lines], np.float32), s.vertices)


def test_fragment_files_and_their_merge(tmp_path):
    seg = tubes((6, 16, 40), 15, 2)
    w, off = (40, 4, 4), (3, 10, 20)
    halves = [(seg[:, :, :20], off), (seg[:, :, 20:], (off[0], off[1], off[2] + 20))]
    frags = tmp_path / "frags"
    for part, o in halves:
        sk = {k: Skeleton(*v) for k, v in S.skeletonize(part, w, const=10, dust_threshold=0).items()}
        names = write_fragments(sk, f"file://{frags}", o, part.shape, w)
        assert names == [f"{k}:{bbox_string(o, part.shape)}" for k in sorted(sk)]
        assert bbox_string(o, part.shape) == f"{o[0]}-{o[0] + 6}_{o[1]}-{o[1] + 16}_{o[2]}-{o[2] + 20}"
    merged = aggregate_fragments(str(frags), str(tmp_path / "out"))
    for k, s in merged.items():
        with open(tmp_path / "out" / str(k), "rb") as f:
            assert Skeleton.from_precomputed(f.read()) == s
        parts = []
        for part, o in halves:
            one = S.skeletonize(part, w, const=10, dust_threshold=0)
            if k in one:
                v, e, r = one[k]
                parts.append(Skeleton(v + (np.asarray(o, np.float64) * w)[::-1].astype(np.float32), e, r))
        assert s == Skeleton.merge(parts)
        assert len(np.unique(s.vertices, axis=0)) == len(s.vertices)
        assert len({tuple(sorted(e)) for e in s.edges.tolist()}) == len(s.edges)


def test_merge_drops_equal_vertices_and_duplicate_edges():
    a = Skeleton([[0, 0, 0], [1, 0, 0], [2, 0, 0]], [[1, 0], [2, 1]], [1, 2, 3])
    b = Skeleton([[2, 0, 0], [1, 0, 0], [3, 0, 0]], [[0, 1], [2, 0]], [5, 6, 7])
    m = Skeleton.merge([a, b])
    assert m.vertices.tolist() == [[0, 0, 0], [1, 0, 0], [2, 0, 0], [3, 0, 0]]
    assert m.edges.tolist() == [[0, 1], [1, 2], [2, 3]]
    assert m.radii.tolist() == [1, 2, 3, 7]


def test_local_paths_only(tmp_path):
    with pytest.raises(ValueError):
        write_fragments({}, "gs://bucket/skeletons", (0, 0, 0), (1, 1, 1), (1, 1, 1))


def test_cli_has_the_reference_options():
    from chunkflow_b200.flow.cli import main
    agg = {o for p in main.commands["aggregate-skeleton-fragments"].params for o in p.opts}
    assert {"-i", "-p", "-f", "-o", "--input-name", "--prefix", "--fragments-path", "--output-path"} <= agg
    sk = {o for p in main.commands["skeletonize"].params for o in p.opts}
    assert {"--name", "-i", "-v", "-o", "-t", "--scale", "--const", "--pdrf-scale", "--pdrf-exponent", "--dust-threshold", "-s"} <= sk


# ---- the geodesic field must stay finite and strictly increasing ----
BOUND_REFUSED = [
    (np.ones((3, 1, 1), np.uint32), (1e200, 1, 1), 1e5),   # the z step is sqrt(1e400) = inf
    (np.ones((3, 4, 5), np.uint32), (1, 1, 1), 1e308),     # pdrf_scale + 1 times a step overflows
    (np.ones((3, 4, 5), np.uint32), (1, 1, 1), 1e17),      # D can reach 2^53: a step no longer raises it
    (np.ones((3, 4, 5), np.uint32), (40, 4, 4), 1e14),
]


@pytest.mark.parametrize("seg, w, pdrf_scale", BOUND_REFUSED)
def test_unbounded_geodesic_fields_are_refused_before_any_kernel(emu, seg, w, pdrf_scale):
    with pytest.raises(ValueError, match="strictly increasing"):
        S.skeletonize(seg, w, pdrf_scale=pdrf_scale, dust_threshold=0)
    with pytest.raises(ValueError, match="strictly increasing"):
        check_params(4, 500, pdrf_scale, 4, 0, w, seg.shape)
    work = np.zeros(N.skeleton_workspace(seg.shape, emu), np.uint8)
    args = (seg.ctypes.data, N.DTYPE_U32, seg.shape, w)
    counts = N.skeleton_count_device(*args, 0, 0, 0, work.ctypes.data, lib=emu)
    buf = np.zeros(counts[2], np.uint8)
    with pytest.raises(N.NativeError, match="strictly increasing") as err:
        N.skeleton_device(*args, 4, 500, pdrf_scale, 4, work.ctypes.data, counts, buf.ctypes.data, lib=emu)
    assert err.value.code == N.ERR_INVALID_ARGUMENT
    if w[0] > 1e100:
        return
    # refused before anything ran: the same count still serves a legal call
    n, _ = N.skeleton_device(*args, 4, 500, 1e5, 4, work.ctypes.data, counts, buf.ctypes.data, lib=emu)
    got = N.skeleton_read(buf.ctypes.data, seg.shape, w, counts, n, lib=emu)
    assert_same(got, S.skeletonize(seg, w, dust_threshold=0))


def test_the_bound_admits_the_defaults_on_the_largest_chunks():
    check_params(4, 500, 100000, 4, 1000, (40, 4, 4), (1024, 2048, 2047))
    check_params(4, 500, 100000, 4, 1000, (1, 1, 1), (1024, 2048, 2047))
    S.check_params(4, 500, 100000, 4, 1000, (40, 4, 4), 2 ** 32 - 1)
    with pytest.raises(ValueError):
        check_params(4, 500, 100000, 4, 1000, (40, 1, 1), (1024, 2048, 2047))


def test_a_count_serves_one_skeleton_call(emu):
    seg = VOLUMES["tubes"]()
    work = np.zeros(N.skeleton_workspace(seg.shape, emu), np.uint8)
    args = (seg.ctypes.data, N.DTYPE_U32, seg.shape, (1, 1, 1))
    counts = N.skeleton_count_device(*args, 0, 0, 0, work.ctypes.data, lib=emu)
    buf = np.zeros(counts[2], np.uint8)
    N.skeleton_device(*args, 1, 2, 1e5, 4, work.ctypes.data, counts, buf.ctypes.data, lib=emu)
    with pytest.raises(N.NativeError, match="one cfb_skeleton_device per cfb_skeleton_count_device"):
        N.skeleton_device(*args, 1, 2, 1e5, 4, work.ctypes.data, counts, buf.ctypes.data, lib=emu)
    counts = N.skeleton_count_device(*args, 0, 0, 0, work.ctypes.data, lib=emu)   # a new count makes it usable again
    n, _ = N.skeleton_device(*args, 1, 2, 1e5, 4, work.ctypes.data, counts, buf.ctypes.data, lib=emu)
    assert_same(N.skeleton_read(buf.ctypes.data, seg.shape, (1, 1, 1), counts, n, lib=emu), S.skeletonize(seg, (1, 1, 1), scale=1, const=2, dust_threshold=0))


def test_the_distance_transform_has_its_own_smaller_workspace(emu):
    seg = VOLUMES["blobs"]()
    assert N.edt_workspace(seg.shape, emu) == 16 * seg.size < N.skeleton_workspace(seg.shape, emu)
    ids = S.as_ids(seg)
    work = np.zeros(N.edt_workspace(ids.shape, emu), np.uint8)
    out = np.zeros(ids.shape, np.float32)
    N.edt_device(ids.ctypes.data, N.DTYPE_U64, ids.shape, (40, 4, 4), out.ctypes.data, work.ctypes.data, lib=emu)
    assert np.array_equal(out, S.distance_transform(seg, (40, 4, 4)))
