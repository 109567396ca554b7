"""`skeletonize` on the GPU: DeviceChunk.distance_transform against live scipy, DeviceChunk.skeletonize against
oracle/skeleton_oracle.py (== on vertices, edges and radii) for every id dtype, a branching-tube volume that needs many sweeps
and rounds, and the `skeletonize` / `aggregate-skeleton-fragments` commands against the oracle's files."""
import os

import numpy as np
import pytest
from scipy import ndimage

from oracle import skeleton_oracle as S

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("the gpu tests need a CUDA device")
    return torch


def blobs(shape, seed, n=6):
    rng = np.random.default_rng(seed)
    z, y, x = np.indices(shape)
    seg = np.zeros(shape, np.uint32)
    for i in range(1, n + 1):
        c, r = rng.uniform(0, shape), rng.uniform(1.5, max(2.0, max(shape) / 3), 3)
        seg[((z - c[0]) / r[0]) ** 2 + ((y - c[1]) / r[1]) ** 2 + ((x - c[2]) / r[2]) ** 2 < 1] = i * 7919
    return seg


def tubes(shape, seed, n=3, radius=2.0, branches=2):
    rng = np.random.default_rng(seed)
    z, y, x = np.indices(shape)
    seg = np.zeros(shape, np.uint32)
    for t in range(1, n + 1):
        cz, cy = rng.uniform(radius, shape[0] - radius), rng.uniform(radius, shape[1] - radius)
        seg[(z - cz) ** 2 + (y - cy) ** 2 <= radius ** 2] = t
        for _ in range(branches):
            bx = rng.uniform(0, shape[2])
            seg[((z - cz) ** 2 + (x - bx) ** 2 <= radius ** 2) & (y > cy)] = t
    return seg


def scipy_dbf(seg, w):
    out = np.zeros(seg.shape, np.float32)
    for L in np.unique(seg):
        if L != 0:
            d = ndimage.distance_transform_edt(np.pad(seg == L, 1), sampling=w)[1:-1, 1:-1, 1:-1].astype(np.float32)
            out[seg == L] = d[seg == L]
    return out


def device_chunk(torch, seg, voxel_size=(1, 1, 1)):
    from chunkflow_b200.chunk.device import DeviceChunk
    arr = np.ascontiguousarray(seg)
    arr = arr.view(np.int32 if arr.itemsize == 4 else np.int64)
    return DeviceChunk(torch.from_numpy(arr).cuda(), voxel_size=voxel_size)


def assert_same(got: dict, want: dict):
    assert list(got) == list(want)
    for k in want:
        v, e, r = want[k]
        assert np.array_equal(got[k].vertices, v) and np.array_equal(got[k].edges, e) and np.array_equal(got[k].radii, r), k


@pytest.mark.parametrize("shape", [(1, 1, 1), (2, 1, 70), (1, 33, 2), (7, 40, 45), (33, 17, 64), (64, 64, 64)])
@pytest.mark.parametrize("w", [(1, 1, 1), (40, 4, 4)])
def test_distance_transform_is_scipy(torch, shape, w):
    rng = np.random.default_rng(sum(shape))
    for seg in (rng.integers(0, 3, shape).astype(np.uint32), blobs(shape, shape[0])):
        got = device_chunk(torch, seg).distance_transform(voxel_size=w).tensor.cpu().numpy()
        assert np.array_equal(got, scipy_dbf(seg, w))


def test_distance_transform_at_non_integer_voxel_sizes_is_the_oracle(torch):
    seg = blobs((12, 30, 34), 4, 10)
    w = (1.5, 0.75, 2.25)
    assert np.array_equal(device_chunk(torch, seg).distance_transform(voxel_size=w).tensor.cpu().numpy(), S.distance_transform(seg, w))


@pytest.mark.parametrize("dtype", ["uint32", "int32", "uint64", "int64"])
def test_skeletonize_equals_the_oracle_for_every_id_dtype(torch, dtype):
    seg = (blobs((12, 26, 28), 3).astype(np.int64) + tubes((12, 26, 28), 5).astype(np.int64) * 100003)
    seg[seg > 0] -= 3 * 7919   # negative ids too: read by their unsigned bit pattern
    seg = seg.astype(dtype)
    skip = [int(seg.flat[np.flatnonzero(seg)[0]])]
    for w, p in [((40, 4, 4), dict(const=20, scale=1, dust_threshold=5)), ((1, 1, 1), dict(const=2, dust_threshold=0)),
                 ((1.5, 0.75, 2.25), dict(const=1, scale=2, pdrf_exponent=7, dust_threshold=10))]:
        got = device_chunk(torch, seg).skeletonize(voxel_size=w, skip_ids=skip, **p)
        assert_same(got, S.skeletonize(seg, w, skip_ids=skip, **p))
        assert (skip[0] % 2 ** 32 if seg.itemsize == 4 else skip[0] % 2 ** 64) not in got


def test_defaults_and_refusals(torch):
    from chunkflow_b200.chunk.device import DeviceChunk
    seg = blobs((16, 40, 40), 6)
    assert_same(device_chunk(torch, seg, (40, 4, 4)).skeletonize(), S.skeletonize(seg, (40, 4, 4)))
    assert device_chunk(torch, np.zeros((3, 4, 5), np.uint32)).skeletonize(dust_threshold=0) == {}
    with pytest.raises(TypeError):
        DeviceChunk(torch.zeros((4, 4, 4), dtype=torch.float32, device="cuda")).skeletonize()
    with pytest.raises(ValueError):
        DeviceChunk(torch.zeros((1, 4, 4, 4), dtype=torch.int32, device="cuda")).skeletonize()
    with pytest.raises(ValueError):
        device_chunk(torch, seg).skeletonize(pdrf_exponent=0)
    for w, pdrf_scale in (((1e200, 1, 1), 1e5), ((1, 1, 1), 1e308), ((1, 1, 1), 1e17)):   # D could overflow or stop growing
        with pytest.raises(ValueError, match="strictly increasing"):
            device_chunk(torch, seg).skeletonize(voxel_size=w, pdrf_scale=pdrf_scale, dust_threshold=0)


def test_branching_tubes_need_many_sweeps_and_rounds(torch):
    seg = tubes((24, 96, 160), 7, 4, 2.5, 5)
    st = {}
    got = device_chunk(torch, seg).skeletonize(voxel_size=(1, 1, 1), const=2, scale=1, dust_threshold=50, stats=st)
    assert st["sweeps"] >= 10 and st["rounds"] >= 5, st
    assert_same(got, S.skeletonize(seg, (1, 1, 1), const=2, scale=1, dust_threshold=50))


def tree(path):
    out = {}
    for d, _, files in os.walk(path):
        for name in files:
            with open(os.path.join(d, name), "rb") as f:
                out[os.path.relpath(os.path.join(d, name), path)] = f.read()
    return out


@pytest.mark.parametrize("to_device", [False, True])
@pytest.mark.parametrize("fmt", ["precomputed", "swc"])
def test_cli_after_connected_components_writes_what_the_oracle_writes(torch, tmp_path, to_device, fmt):
    from chunkflow_b200.chunk import Chunk
    from chunkflow_b200.flow.cli import main
    from chunkflow_b200.flow.skeleton import Skeleton, write_fragments
    mine, theirs = tmp_path / "mine", tmp_path / "theirs"
    args = ["create-chunk", "--size", "8", "48", "48", "--pattern", "sin", "--voxel-offset", "2", "10", "20", "--voxel-size", "40", "4", "4",
            "connected-components", "--threshold", "0.5"]
    args += ["to-device"] if to_device else []
    args += ["skeletonize", "-o", f"file://{mine}", "-t", fmt, "--const", "40", "--scale", "2", "--dust-threshold", "20", "-s", "1"]
    tasks = main.main(args, standalone_mode=False)
    seg = tasks[0]["chunk"]
    assert isinstance(seg, Chunk) != to_device
    arr = seg.to_chunk().array if to_device else seg.array
    want = {k: Skeleton(*v) for k, v in S.skeletonize(arr, (40, 4, 4), const=40, scale=2, dust_threshold=20, skip_ids=[1]).items()}
    assert want
    write_fragments(want, str(theirs), (2, 10, 20), arr.shape, (40, 4, 4), fmt)
    assert tree(str(mine)) == tree(str(theirs))


def test_aggregate_over_two_chunks_writes_what_the_oracle_merges(torch, tmp_path):
    from chunkflow_b200.chunk import Chunk
    from chunkflow_b200.flow.cli import main
    from chunkflow_b200.flow.skeleton import Skeleton
    seg = tubes((8, 40, 64), 9, 3, 2.0)
    frags = tmp_path / "frags"
    parts = [(seg[:, :, :32], (0, 0, 0)), (seg[:, :, 32:], (0, 0, 32))]
    for part, off in parts:
        tasks = [{"log": {"timer": {}}, "chunk": Chunk(np.ascontiguousarray(part), voxel_offset=off, voxel_size=(40, 4, 4))}]
        op = main.commands["skeletonize"].callback(name="skeletonize", input_chunk_name="chunk", voxel_size=None, output_path=str(frags),
                                                   output_format="precomputed", scale=2, const=40, pdrf_scale=100000, pdrf_exponent=4,
                                                   dust_threshold=10, skip_ids=None)
        list(op(iter(tasks)))
    from chunkflow_b200.flow.skeleton import aggregate_fragments
    op = main.commands["aggregate-skeleton-fragments"].callback(name="aggregate-skeleton-fragments", input_name="prefix", prefix=None,
                                                                fragments_path=str(frags), output_path=str(tmp_path / "out"))
    list(op(iter([{"log": {"timer": {}}, "prefix": ""}])))
    got = tree(str(tmp_path / "out"))
    ids = sorted({int(n.split(":")[0]) for n in os.listdir(frags)})
    assert sorted(got) == [str(i) for i in ids] and len(ids) >= 2
    for i in ids:
        pieces = []
        for part, off in parts:
            one = S.skeletonize(part, (40, 4, 4), const=40, scale=2, dust_threshold=10)
            if i in one:
                v, e, r = one[i]
                pieces.append(Skeleton(v + (np.asarray(off, np.float64) * (40, 4, 4))[::-1].astype(np.float32), e, r))
        assert got[str(i)] == Skeleton.merge(pieces).to_precomputed()
    assert aggregate_fragments(str(frags), str(tmp_path / "again")).keys() == set(ids)
