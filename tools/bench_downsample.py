"""Benchmark of `downsample` on the GPU (csrc/downsample.cu): one JSON line.

    python tools/bench_downsample.py [--sizes 512 1024] [--iters 5]

Cases: cubes of 512^3 and 1024^3 voxels; uint8 images (random values) with (2,2,2) and (1,2,2), which take the vectorised
kernel (16-byte loads), and with (4,4,4) and (2,2,1), which take the generic one; uint32 and uint64 labels,
"blobs" (coherent 16 x 32 x 32 blocks of one id each: the common case of a segmentation) and "salt" (every voxel an independent
random id of 10^6: no two voxels of a block agree), with (2,2,2), (1,2,2) and (4,4,4) -- one, one and two countless levels.

Per case: the kernels alone (cfb_downsample_average_device / cfb_downsample_segmentation_device into preallocated buffers) and
DeviceChunk.downsample end to end (plan, allocation of output and workspace), CUDA events, mean of --iters after a warm-up.
Algorithmic bytes -- the input read once and every level written once -- over the kernel time, as a share of the 3.35 TB/s
HBM3 figure of the H100 SXM data sheet (a data-sheet figure, not a measured one).  The device name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip() or "not available"
    except Exception:
        return "not available"


def make_volume(torch, size, kind, dtype):
    g = torch.Generator(device="cuda").manual_seed(0)
    if kind == "image":
        return torch.randint(0, 256, (size, size, size), device="cuda", generator=g, dtype=torch.uint8)
    if kind == "blobs":
        z = torch.arange(size, device="cuda", dtype=torch.int64).view(-1, 1, 1)
        y = torch.arange(size, device="cuda", dtype=torch.int64).view(1, -1, 1)
        x = torch.arange(size, device="cuda", dtype=torch.int64).view(1, 1, -1)
        seg = ((z // 16) * 1_000_003 + (y // 32) * 1009 + (x // 32)).expand(size, size, size)
    else:
        seg = torch.randint(0, 1_000_000, (size, size, size), device="cuda", generator=g, dtype=torch.int64)
    if dtype == "uint64":   # spread the ids over the whole 64-bit range (an odd multiplier is a bijection modulo 2^64)
        return (seg * -7046029254386353131).contiguous()
    return seg.to(torch.int32).contiguous()


def timed(torch, iters, fn):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    total = 0.0
    for _ in range(iters):
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        total += e0.elapsed_time(e1)
    return total / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[512, 1024])
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    import torch
    from chunkflow_b200 import _native
    from chunkflow_b200.chunk.device import DeviceChunk
    if not torch.cuda.is_available():
        raise SystemExit("bench_downsample needs a CUDA device")
    stream = torch.cuda.current_stream().cuda_stream
    share = lambda nbytes, ms: round(nbytes / (ms * 1e-3) / HBM_PEAK, 3)
    cases = []
    plan = [("image", "uint8", f) for f in ((2, 2, 2), (1, 2, 2), (4, 4, 4), (2, 2, 1))]
    plan += [(kind, dtype, f) for dtype in ("uint32", "uint64") for kind in ("blobs", "salt") for f in ((2, 2, 2), (1, 2, 2), (4, 4, 4))]
    for size in args.sizes:
        volumes = {}
        for kind, dtype, f in plan:
            key = (kind, dtype)
            if key not in volumes:
                volumes.clear()
                torch.cuda.empty_cache()
                volumes[key] = make_volume(torch, size, kind, dtype)
            t = volumes[key]
            width = t.element_size()
            if kind == "image":
                out_shape, work_bytes, levels = tuple(-(-size // k) for k in f), 0, [tuple(-(-size // k) for k in f)]
                out = torch.empty(out_shape, dtype=t.dtype, device="cuda")
                kernel = lambda: _native.downsample_average_device(t.data_ptr(), t.shape, f, out.data_ptr(), stream)
            else:
                code = _native.DTYPE_U64 if dtype == "uint64" else _native.DTYPE_U32
                out_shape, work_bytes = _native.downsample_workspace(code, t.shape, f)
                levels = [tuple(size // 2 ** (i + 1) if k > 1 else size for k in (min(v, 2) for v in f))
                          for i in range(1 if max(f) <= 2 else 2)]
                out = torch.empty(out_shape, dtype=t.dtype, device="cuda")
                work = torch.empty(max(work_bytes, 1), dtype=torch.uint8, device="cuda")
                kernel = lambda: _native.downsample_segmentation_device(t.data_ptr(), code, t.shape, f, work.data_ptr(), out.data_ptr(),
                                                                        stream)
            nbytes = t.numel() * width + sum(a * b * c for a, b, c in levels) * width
            kernel_ms = timed(torch, args.iters, kernel)
            e2e_ms = timed(torch, args.iters, lambda: DeviceChunk(t).downsample(f))
            path = ("vectorised" if f[1:] == (2, 2) and f[0] <= 2 else "generic") if kind == "image" else "generic"
            cases.append(dict(size=size, kind=kind, dtype=dtype, factor=list(f), path=path, output=list(out_shape), levels=len(levels),
                              workspace_bytes=work_bytes, kernel_ms=round(kernel_ms, 3),
                              kernel_share_of_hbm_peak=share(nbytes, kernel_ms), algorithmic_bytes=nbytes,
                              device_chunk_downsample_ms=round(e2e_ms, 3)))
            del out
            work = None
        volumes.clear()
        torch.cuda.empty_cache()
    print(json.dumps({"bench": "downsample", "device": torch.cuda.get_device_name(0), "power_limit": power_limit(),
                      "hbm_peak_datasheet_tb_s": 3.35, "timing": "CUDA events, mean of %d after a warm-up" % args.iters,
                      "cases": cases}))


if __name__ == "__main__":
    main()
