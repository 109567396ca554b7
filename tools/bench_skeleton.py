"""Benchmark of `skeletonize` on the GPU (csrc/skeleton.cu): one JSON line.

    python tools/bench_skeleton.py [--sizes 512 1024] [--iters 1]

Cases: cubes of 512^3 and 1024^3 int32 ids.  "blobs" are bench_relabel.py's coherent 16 x 32 x 32 blocks of one id each, at a
(40, 4, 4) nm voxel size with the default parameters (every block is one object).  "tubes" is a sparse volume of branching tubes
(64 trees of radius 4 voxels, each a trunk along x with 6 branches along y) at (1, 1, 1) with const 8, so that every tree takes
several rounds.

Per case: the distance transform alone (cfb_edt_device, CUDA events after a warm-up) and its algorithmic bytes -- the ids read
once and the float32 map written once -- over its time, as a share of the 3.35 TB/s HBM3 peak of the H100 SXM data sheet (a
data-sheet figure, not a measured one); then DeviceChunk.skeletonize end to end (CUDA events) with the relaxation sweeps and
their time, the time of the sort, the rounds, the mean path length, the time of the rounds and, within it, of the serial trace
kernels alone, as cfb_skeleton_device reports them (host clock around work that ends in a synchronise; each round's trace starts
on an idle stream).  A case that does not fit in device memory is reported as such.  The device name
and power limit are read in the same run.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_relabel import HBM_PEAK, make_labels, power_limit, timed  # noqa: E402


def make_tubes(torch, size, trees=64, radius=4, branches=6):
    g = torch.Generator(device="cpu").manual_seed(0)
    seg = torch.zeros((size, size, size), dtype=torch.int32, device="cuda")
    z = torch.arange(size, device="cuda").view(-1, 1, 1)
    y = torch.arange(size, device="cuda").view(1, -1, 1)
    x = torch.arange(size, device="cuda").view(1, 1, -1)
    for t in range(1, trees + 1):
        cz, cy = (torch.rand(2, generator=g) * (size - 2 * radius) + radius).tolist()
        seg[((z - cz) ** 2 + (y - cy) ** 2 <= radius ** 2).expand(size, size, size)] = t
        for bx in (torch.rand(branches, generator=g) * size).tolist():
            m = ((z - cz) ** 2 + (x - bx) ** 2 <= radius ** 2) & (y > cy)
            seg[m.expand(size, size, size)] = t
    return seg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[512, 1024])
    ap.add_argument("--iters", type=int, default=1)
    args = ap.parse_args()
    import torch
    from chunkflow_b200 import _native as N
    from chunkflow_b200.chunk.device import DeviceChunk
    cases = []
    for size in args.sizes:
        for kind in ("blobs", "tubes"):
            case = {"size": size, "kind": kind}
            try:
                seg = make_labels(torch, size, "blobs", False) if kind == "blobs" else make_tubes(torch, size)
                vs, kw = ((40, 4, 4), {}) if kind == "blobs" else ((1, 1, 1), dict(const=8))
                zyx = tuple(seg.shape)
                out = torch.empty(zyx, dtype=torch.float32, device="cuda")
                work = torch.empty(N.edt_workspace(zyx), dtype=torch.uint8, device="cuda")
                edt_ms = timed(torch, 3, lambda: N.edt_device(seg.data_ptr(), N.DTYPE_U32, zyx, vs, out.data_ptr(), work.data_ptr()))
                del work, out
                torch.cuda.empty_cache()
                nbytes = seg.numel() * (4 + 4)
                case.update(edt_ms=round(edt_ms, 3), edt_hbm_share=round(nbytes / (edt_ms * 1e-3) / HBM_PEAK, 4))
                dev, st = DeviceChunk(seg, voxel_size=vs), {}
                e2e = timed(torch, args.iters, lambda: dev.skeletonize(stats=st, **kw))
                skels = dev.skeletonize(**kw)
                case.update(end_to_end_ms=round(e2e, 1), objects=len(skels), sweeps=int(st["sweeps"]), relax_ms=round(st["relax_ms"], 1),
                            sort_ms=round(st["sort_ms"], 1), rounds=int(st["rounds"]), paths=int(st["paths"]),
                            mean_path_length=round(st["skeleton_voxels"] / max(st["paths"], 1), 2), rounds_ms=round(st["rounds_ms"], 1),
                            trace_ms=round(st["trace_ms"], 1), vertices=int(st["skeleton_voxels"]))
                del dev, seg, skels
            except (torch.cuda.OutOfMemoryError, RuntimeError) as exc:
                case["not_measured"] = str(exc).splitlines()[0][:200]
            torch.cuda.empty_cache()
            print(json.dumps(case), file=sys.stderr, flush=True)
            cases.append(case)
    print(json.dumps({"bench": "skeleton", "device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "cases": cases}))


if __name__ == "__main__":
    main()
