"""`mesh` on the GPU: DeviceChunk.mesh against oracle/mesh_oracle.py (== on vertices and faces, unsimplified and simplified) and
the `mesh` command after create-chunk -> connected-components, on host and GPU-resident chunks, against the oracle's writer."""
import os

import numpy as np
import pytest

from oracle import mesh_oracle as M

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("the gpu tests need a CUDA device")
    return torch


def blobs(shape, seed, n=8):
    rng = np.random.default_rng(seed)
    z, y, x = np.indices(shape)
    seg = np.zeros(shape, np.uint32)
    for i in range(1, n + 1):
        c, r = rng.uniform(0, shape), rng.uniform(1.5, max(2.0, max(shape) / 3), 3)
        seg[((z - c[0]) / r[0]) ** 2 + ((y - c[1]) / r[1]) ** 2 + ((x - c[2]) / r[2]) ** 2 < 1] = i * 7919
    return seg


def assert_same(a: dict, b: dict):
    assert list(a) == list(b)
    for k in a:
        assert np.array_equal(a[k][0], b[k][0]) and np.array_equal(a[k][1], b[k][1]), k


def device_chunk(torch, seg, voxel_size=(40, 4, 4)):
    from chunkflow_b200.chunk.device import DeviceChunk
    t = torch.from_numpy(np.ascontiguousarray(seg)).cuda()
    return DeviceChunk(t, voxel_size=voxel_size)


GEOMETRIES = [(1, 1, 1), (1, 8, 9), (2, 2, 2), (3, 1, 17), (5, 6, 7), (8, 33, 31), (17, 16, 15), (4, 64, 64), (32, 40, 24),
              (2, 100, 3), (9, 9, 70), (24, 24, 24)]


@pytest.mark.parametrize("shape", GEOMETRIES)
def test_device_mesh_equals_the_oracle(torch, shape):
    rng = np.random.default_rng(sum(shape))
    for seg in (rng.integers(0, 5, shape).astype(np.uint32), blobs(shape, len(shape) + shape[0])):
        for close in (False, True):
            got = device_chunk(torch, seg).mesh(simplification_factor=1, close=close)
            assert_same(got, M.marching_cubes(seg, (40, 4, 4), close=close))


@pytest.mark.parametrize("dtype", ["uint32", "int32", "uint64", "int64"])
def test_every_id_dtype_and_skip_ids(torch, dtype):
    seg = blobs((12, 30, 28), 3).astype(np.int64)
    seg[seg > 0] -= 3 * 7919   # negative ids too: read by their unsigned bit pattern
    seg = seg.astype(dtype)
    tdt = {"uint32": torch.int32, "int32": torch.int32, "uint64": torch.int64, "int64": torch.int64}[dtype]
    from chunkflow_b200.chunk.device import DeviceChunk
    t = torch.from_numpy(seg.view(np.int32 if seg.itemsize == 4 else np.int64)).cuda().to(tdt)
    skip = [int(seg.flat[np.flatnonzero(seg)[0]])]
    for close in (False, True):
        got = DeviceChunk(t, voxel_size=(8, 6, 5)).mesh(simplification_factor=1, skip_ids=skip, close=close)
        assert_same(got, M.marching_cubes(seg, (8, 6, 5), skip_ids=skip, close=close))
        assert len(got) == len(np.unique(seg[seg != 0])) - 1


def test_simplified_meshes_equal_the_oracle(torch):
    seg = blobs((12, 24, 24), 11, 4)
    for close in (False, True):
        for factor, err in ((100, 40), (10, 8), (4, 1000)):
            got = device_chunk(torch, seg).mesh(simplification_factor=factor, max_simplification_error=err, close=close, threads=3)
            want = {k: M.simplify(v, f, factor, err) for k, (v, f) in M.marching_cubes(seg, (40, 4, 4), close=close).items()}
            assert_same(got, want)


def test_a_non_contiguous_view(torch):
    from chunkflow_b200.chunk.device import DeviceChunk
    seg = blobs((10, 30, 40), 5)
    t = torch.from_numpy(seg.view(np.int32)).cuda().permute(0, 2, 1)[:, 3:35:2, 1:]
    assert not t.is_contiguous()
    want = M.marching_cubes(t.cpu().numpy().view(np.uint32), (1, 1, 1), close=True)
    assert_same(DeviceChunk(t).mesh(simplification_factor=1, close=True), want)


def test_refusals(torch):
    from chunkflow_b200.chunk.device import DeviceChunk
    with pytest.raises(TypeError):
        DeviceChunk(torch.zeros((4, 4, 4), dtype=torch.float32, device="cuda")).mesh()
    with pytest.raises(TypeError):
        DeviceChunk(torch.zeros((4, 4, 4), dtype=torch.uint8, device="cuda")).mesh()
    with pytest.raises(ValueError):
        DeviceChunk(torch.zeros((1, 4, 4, 4), dtype=torch.int32, device="cuda")).mesh()


def tree(path):
    out = {}
    for d, _, files in os.walk(path):
        for name in files:
            with open(os.path.join(d, name), "rb") as f:
                out[os.path.relpath(os.path.join(d, name), path)] = f.read()
    return out


@pytest.mark.parametrize("to_device", [False, True])
@pytest.mark.parametrize("fmt, extra", [("obj", []), ("ply", []), ("precomputed", []), ("precomputed", ["--manifest"]),
                                        ("precomputed", ["--shard"])])
def test_cli_after_connected_components_writes_what_the_oracle_writes(torch, tmp_path, to_device, fmt, extra):
    import json
    from chunkflow_b200.chunk import Chunk
    from chunkflow_b200.flow.cli import main
    mine, theirs = tmp_path / "mine", tmp_path / "theirs"
    for p in (mine, theirs):
        os.makedirs(p)
        if fmt == "precomputed":
            with open(p / "info", "w") as f:
                json.dump({"scales": [{"resolution": [4, 4, 40]}]}, f)
    args = ["create-chunk", "--size", "4", "24", "24", "--pattern", "sin", "--voxel-offset", "2", "10", "20", "--voxel-size", "40", "4", "4",
            "connected-components", "--threshold", "0.5"]
    args += ["to-device"] if to_device else []
    args += ["mesh", "-o", f"file://{mine}", "-t", fmt, "-f", "10", "-e", "40", "-s", "1"] + extra
    tasks = main.main(args, standalone_mode=False)
    seg = tasks[0]["chunk"]
    assert isinstance(seg, Chunk) != to_device
    arr = seg.to_chunk().array if to_device else seg.array
    meshes = {k: M.simplify(v, f, 10, 40) for k, (v, f) in M.marching_cubes(arr, (40, 4, 4),
                                                                             skip_ids=() if "--shard" in extra else (1,)).items()}
    M.write(meshes, str(theirs), fmt, (2, 10, 20), arr.shape, (40, 4, 4), manifest="--manifest" in extra, shard="--shard" in extra,
            skip_ids={1})
    a, b = tree(str(mine)), tree(str(theirs))
    assert len(a) > 2 and a == b
