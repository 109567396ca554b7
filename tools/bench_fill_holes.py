"""Benchmark of `fill-segmentation-holes` on the GPU (csrc/fill_holes.cu): one JSON line.

    python tools/bench_fill_holes.py [--sizes 512 1024] [--salt-sizes 256] [--iters 3]

Inputs:
  * "blocks": bench_relabel.py's coherent 16 x 32 x 32 blocks of one id each (int32), with a cavity of 8 x 16 x 16 zeros carved
    in every block and, in every eighth block, an inner object of 4 x 8 x 8 voxels with a gap of zeros around it.  Run in both
    per-object modes and in binary mode.
  * "balls": a binary uint8 volume of hollow balls (one per 64^3 cell, shell radii 17 to 20): binary mode.
  * "salt": salt-and-pepper ids, every voxel an independent draw from 0..3 (int32), at --salt-sizes: every mode.

Per case: DeviceChunk.fill_holes end to end (CUDA events after a warm-up, mean of --iters), then one call's phases --
components (union-find, flatten, scan, numbering, faces), graph (the pair table, grown on overflow), host enclosure (gather,
copy, Hopcroft-Tarjan, map upload) and apply -- as the host clock around synchronised calls, with the components, pairs and
table slots.  Rates: the streaming bytes of the voxel passes (each input, workspace or output array read or written once per
pass; the gathers through the union-find and the component map are not counted) over the time of their phase, as a share of
the 3.35 TB/s HBM3 figure of the H100 SXM data sheet (a data-sheet figure, not a measured one).  A case that does not fit is
reported with the refusal's message.  The device name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_relabel import HBM_PEAK, power_limit, timed  # noqa: E402


def make_blocks(torch, size):
    z = torch.arange(size, device="cuda", dtype=torch.int64).view(-1, 1, 1)
    y = torch.arange(size, device="cuda", dtype=torch.int64).view(1, -1, 1)
    x = torch.arange(size, device="cuda", dtype=torch.int64).view(1, 1, -1)
    block = (z // 16) * 1_000_003 + (y // 32) * 1009 + (x // 32)
    lz, ly, lx = z % 16, y % 32, x % 32
    cavity = (lz >= 4) & (lz < 12) & (ly >= 8) & (ly < 24) & (lx >= 8) & (lx < 24)
    inner = (lz >= 6) & (lz < 10) & (ly >= 12) & (ly < 20) & (lx >= 12) & (lx < 20) & (block % 8 == 0)
    seg = torch.where(cavity, torch.where(inner, block + (1 << 30), 0), block + 1)
    return seg.expand(size, size, size).to(torch.int32).contiguous()


def make_balls(torch, size, cell=64):
    c = (torch.arange(size, device="cuda") % cell - (cell - 1) / 2) ** 2
    r2 = c.view(-1, 1, 1) + c.view(1, -1, 1) + c.view(1, 1, -1)
    return ((r2 >= 17 ** 2) & (r2 <= 20 ** 2)).to(torch.uint8).contiguous()


def make_salt(torch, size):
    g = torch.Generator(device="cuda").manual_seed(0)
    return torch.randint(0, 4, (size, size, size), device="cuda", generator=g, dtype=torch.int32)


def pass_bytes(n, item, binary):
    """Streaming bytes of each phase's voxel passes (see the module doc)."""
    seg = n * item
    components = (4 * n                       # init: P written
                  + seg + 4 * n               # merge: ids and P read
                  + 3 * 4 * n                 # flatten: P read and written, root flags written
                  + 3 * 4 * n                 # scan: the flags read twice, the ranks written
                  + 3 * 4 * n                 # numbering: P and ranks read, components written
                  + (2 * seg if binary else 0))   # binary: the flatten and the numbering read the ids
    return {"components": components, "graph": 0 if binary else 4 * n, "apply": 2 * seg + 4 * n}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[512, 1024])
    ap.add_argument("--salt-sizes", type=int, nargs="+", default=[256])
    ap.add_argument("--iters", type=int, default=3)
    args = ap.parse_args()
    import torch
    from chunkflow_b200.chunk.device import DeviceChunk
    plan = [(s, k, m) for s in args.sizes for k, modes in (("blocks", ("keep-enclosed", "remove-enclosed", "binary")), ("balls", ("binary",)))
            for m in modes]
    plan += [(s, "salt", m) for s in args.salt_sizes for m in ("binary", "keep-enclosed", "remove-enclosed")]
    cases, cache = [], {}
    for size, kind, mode in plan:
        case = {"size": size, "kind": kind, "mode": mode}
        try:
            if (size, kind) not in cache:
                cache.clear()
                torch.cuda.empty_cache()
                cache[(size, kind)] = {"blocks": make_blocks, "balls": make_balls, "salt": make_salt}[kind](torch, size)
            seg = cache[(size, kind)]
            dev = DeviceChunk(seg)
            e2e = timed(torch, args.iters, lambda: dev.fill_holes(mode))
            st = {}
            _, count = dev.fill_holes(mode, return_fill_count=True, stats=st)
            nb = pass_bytes(seg.numel(), seg.element_size(), mode == "binary")
            case.update(end_to_end_ms=round(e2e, 1), fill_count=count, components=st["components"], edges=st["edges"],
                        table_slots=st["table_slots"])
            for phase in ("components", "graph", "enclose", "apply"):
                if phase + "_ms" in st:
                    case[phase + "_ms"] = round(st[phase + "_ms"], 2)
                    if nb.get(phase):
                        case[phase + "_hbm_share"] = round(nb[phase] / (st[phase + "_ms"] * 1e-3) / HBM_PEAK, 4)
            del dev
        except (torch.cuda.OutOfMemoryError, RuntimeError) as exc:
            case["not_measured"] = str(exc).splitlines()[0][:300]
        torch.cuda.empty_cache()
        print(json.dumps(case), file=sys.stderr, flush=True)
        cases.append(case)
    print(json.dumps({"bench": "fill_holes", "device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "cases": cases}))


if __name__ == "__main__":
    main()
