"""Benchmark of `mesh` (csrc/mesh.cu): one JSON line.

    python tools/bench_mesh.py [--sizes 256 512 1024] [--host-max-size 256] [--iters 3] [--threads N]

Cases: the coherent segmentations of tools/bench_relabel.py (16 x 32 x 32 blocks of one id each) at every size, uint32 and
uint64 ids, and a sparse one at every size (a few large balls in zeros).  Per case:
  * marching cubes + weld on the device (count, emit, sort by object, weld, place), timed with CUDA events after a warm-up;
    the volume read once over that time, as a share of the 3.35 TB/s HBM3 of the H100 SXM data sheet (a data-sheet figure,
    not a measured one); objects, (cube, object) pairs, triangles, vertices and the device buffer;
  * up to --host-max-size (the host simplifier of a 512^3 chunk of 16 x 32 x 32 blocks, 6.4e7 triangles, takes minutes):
  * the copy of the finished meshes to the host (wall clock);
  * the simplifier at the CLI's defaults (-f 100 -e 40) on N threads over every object, and on 1 thread over the first objects
    (its per-face rate is reported, so that the two can be compared);
  * for the sparse volume, DeviceChunk.mesh plus the writer end to end for each format (precomputed, obj, ply), into a
    temporary directory.
Host steps run for uint32 ids only, after every device case.
The device name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_relabel import HBM_PEAK, make_labels, power_limit, timed  # noqa: E402


def sparse(torch, size):
    z = torch.arange(size, device="cuda", dtype=torch.int64).view(-1, 1, 1)
    y = torch.arange(size, device="cuda", dtype=torch.int64).view(1, -1, 1)
    x = torch.arange(size, device="cuda", dtype=torch.int64).view(1, 1, -1)
    seg = torch.zeros((size, size, size), dtype=torch.int32, device="cuda")
    for i, (cz, cy, cx) in enumerate([(0.3, 0.3, 0.3), (0.7, 0.3, 0.6), (0.5, 0.7, 0.4), (0.25, 0.75, 0.75)]):
        r = 0.18 * size
        ball = (z - cz * size) ** 2 + (y - cy * size) ** 2 + (x - cx * size) ** 2 < r * r
        seg[ball] = i + 1
    return seg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[256, 512, 1024])
    ap.add_argument("--host-max-size", type=int, default=256, help="largest size whose host steps are timed")
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 1)
    ap.add_argument("--serial-objects", type=int, default=200, help="objects simplified on one thread")
    args = ap.parse_args()
    import torch
    from chunkflow_b200 import _native
    from chunkflow_b200.chunk.device import DeviceChunk
    from chunkflow_b200.flow.mesh import MeshWriter
    if not torch.cuda.is_available():
        raise SystemExit("bench_mesh needs a CUDA device")
    stream = torch.cuda.current_stream().cuda_stream
    cases = []
    # every device case first; the host steps (uint32 only) last, the slow simplifier of the blocks without the writers
    plan = [(s, "blobs", w) for s in args.sizes for w in (False, True)] + [(s, "sparse", False) for s in args.sizes]
    plan.sort(key=lambda c: (c[0] <= args.host_max_size and not c[2], c[1] == "sparse"))
    for size, kind, wide in plan:
        seg = sparse(torch, size) if kind == "sparse" else make_labels(torch, size, "blobs", wide)
        code = _native.DTYPE_U64 if wide else _native.DTYPE_U32
        zyx, n, width = tuple(seg.shape), seg.numel(), seg.element_size()
        vs = (40.0, 8.0, 8.0)
        work = torch.empty(_native.mesh_workspace(zyx, False), dtype=torch.uint8, device="cuda")
        a = (seg.data_ptr(), code, zyx, 0, 0, False)
        counts = _native.mesh_count_device(*a, work.data_ptr(), stream)
        pairs, tris, verts = counts
        nbytes = _native.mesh_buffer_bytes(counts)
        buf = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        found = {}

        def device_pass():   # marching cubes + weld: count, emit, sort, weld, place
            c = _native.mesh_count_device(*a, work.data_ptr(), stream)
            found["objects"] = _native.mesh_device(*a, vs, work.data_ptr(), c, buf.data_ptr(), nbytes, stream)

        pass_ms = timed(torch, args.iters, device_pass)
        case = dict(size=size, kind=kind, dtype="uint64" if wide else "uint32", voxels=n, objects=found["objects"], pairs=pairs,
                    triangles=tris, vertices=verts, device_buffer_bytes=nbytes, marching_cubes_and_weld_ms=round(pass_ms, 3),
                    volume_read_share_of_hbm_peak=round(n * width / (pass_ms * 1e-3) / HBM_PEAK, 3))
        cases.append(case)
        print(json.dumps(case), file=sys.stderr, flush=True)
        if size > args.host_max_size or wide:
            del seg, buf, work
            torch.cuda.empty_cache()
            continue
        t0 = time.perf_counter()
        meshes = _native.mesh_read(buf.data_ptr(), counts, found["objects"], stream)
        read_s = time.perf_counter() - t0
        del buf, work
        keys = list(meshes)
        from concurrent.futures import ThreadPoolExecutor
        t0 = time.perf_counter()
        with ThreadPoolExecutor(max_workers=args.threads) as pool:
            simplified = list(pool.map(lambda k: _native.mesh_simplify_host(*meshes[k], 100, 40), keys))
        simplify_n_s = time.perf_counter() - t0
        serial = keys[:args.serial_objects]
        t0 = time.perf_counter()
        for k in serial:
            _native.mesh_simplify_host(*meshes[k], 100, 40)
        simplify_1_s = time.perf_counter() - t0
        serial_faces = sum(len(meshes[k][1]) for k in serial)
        e2e = {}
        chunk = DeviceChunk(seg, voxel_size=vs)
        for fmt in ("precomputed", "obj", "ply") if kind == "sparse" else ():
            with tempfile.TemporaryDirectory() as d:
                if fmt == "precomputed":
                    with open(os.path.join(d, "info"), "w") as f:
                        json.dump({"scales": [{"resolution": list(vs[::-1])}]}, f)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                w = MeshWriter(d, fmt, voxel_size=vs)
                w.write(chunk.mesh(voxel_size=vs, threads=args.threads), (0, 0, 0), zyx)
                e2e[fmt] = round(time.perf_counter() - t0, 3)
        case.update(dict(simplified_triangles=sum(len(f) for _, f in simplified), meshes_to_host_s=round(read_s, 3),
                          simplify_n_threads_s=round(simplify_n_s, 3),
                          simplify_1_thread_us_per_face=round(simplify_1_s / max(serial_faces, 1) * 1e6, 3),
                          simplify_n_threads_us_per_face=round(simplify_n_s / max(tris, 1) * 1e6, 3),
                          end_to_end_s=e2e))
        del seg, chunk, meshes, simplified
        torch.cuda.empty_cache()
        print(json.dumps(case), file=sys.stderr, flush=True)
    print(json.dumps({"bench": "mesh", "device": torch.cuda.get_device_name(0), "power_limit": power_limit(),
                      "host_threads": args.threads, "hbm_peak_datasheet_tb_s": 3.35,
                      "timing": "marching cubes + weld: CUDA events, mean of %d after a warm-up; host steps and end to end: wall clock" % args.iters,
                      "cases": cases}))


if __name__ == "__main__":
    main()
