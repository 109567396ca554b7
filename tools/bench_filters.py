"""Benchmark of `gaussian-filter` and the median filter on the GPU (csrc/filters.cu): one JSON line.

    python tools/bench_filters.py [--sizes 512 1024] [--iters 5]

Cases: cubes of 512^3 and 1024^3 voxels of random values; the gaussian of uint8 and float32 (z,y,x) images with sigma 1 and 2
(radius 4 and 8: two passes per section), and of a float32 (3,z,y,x) affinity map through the command with sigma 1 (three
passes, the channel pass included); the median with (3,1,1) -- the z walk -- and (1,3,3) and (3,3,3) -- the register-window
kernel -- on uint8 and float32.

Per case: the kernels alone (cfb_gaussian_filter_device / cfb_median_filter_device on preallocated buffers), CUDA events, mean
of --iters after a warm-up.  Algorithmic bytes are one read and one write of the chunk; FP64 operations are 3 r + 1 per element
and pass (the multiplies and adds scipy's order needs, each rounded on its own, so no FMA and no tensor cores).  Each is shown
as a share of the H100 SXM data-sheet figure -- 3.35 TB/s of HBM3, 34 TFLOP/s of FP64 without tensor cores -- and the larger
share names the bound.  These are data-sheet figures, not measured ones.  The device name and power limit are read in the same
run.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12
FP64_PEAK = 34e12


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip() or "not available"
    except Exception:
        return "not available"


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
    from chunkflow_b200.chunk.device import gaussian_weights
    if not torch.cuda.is_available():
        raise SystemExit("bench_filters needs a CUDA device")
    stream = torch.cuda.current_stream().cuda_stream
    codes = {"uint8": _native.DTYPE_U8, "float32": _native.DTYPE_F32}
    plan = [("gaussian", dt, 1, s) for dt in ("uint8", "float32") for s in (1, 2)] + [("gaussian", "float32", 3, 1)]
    plan += [("median", dt, 1, size) for dt in ("uint8", "float32") for size in ((3, 1, 1), (1, 3, 3), (3, 3, 3))]
    cases = []
    for size in args.sizes:
        for op, dtype, channels, param in plan:
            torch.cuda.empty_cache()
            shape = (size,) * 3 if channels == 1 else (channels,) + (size,) * 3
            g = torch.Generator(device="cuda").manual_seed(0)
            if dtype == "uint8":
                t = torch.randint(0, 256, shape, device="cuda", generator=g, dtype=torch.uint8)
            else:
                t = torch.rand(shape, device="cuda", generator=g, dtype=torch.float32)
            nbytes = 2 * t.numel() * t.element_size()
            case = dict(size=size, op=op, dtype=dtype, shape=list(shape))
            if op == "gaussian":
                w = gaussian_weights(param)
                weights = [w] * (len(shape) - 1)
                work_bytes = _native.gaussian_filter_workspace(codes[dtype], shape)
                work = torch.empty(work_bytes, dtype=torch.uint8, device="cuda")
                kernel = lambda: _native.gaussian_filter_device(t.data_ptr(), codes[dtype], shape, weights, work.data_ptr(), work_bytes,
                                                                stream)
                flops = t.numel() * len(weights) * (3 * (len(w) - 1) + 1)
                case.update(sigma=param, radius=len(w) - 1, passes=len(weights), workspace_bytes=work_bytes)
            else:
                out = torch.empty_like(t)
                kernel = lambda: _native.median_filter_device(t.data_ptr(), codes[dtype], shape, param, "reflect", out.data_ptr(), stream)
                flops = 0
                case.update(window=list(param), path="z walk" if param == (3, 1, 1) else "register window")
            ms = timed(torch, args.iters, kernel)
            hbm, fp64 = nbytes / (ms * 1e-3) / HBM_PEAK, flops / (ms * 1e-3) / FP64_PEAK
            case.update(kernel_ms=round(ms, 3), algorithmic_bytes=nbytes, fp64_ops=flops, share_of_hbm_peak=round(hbm, 3),
                        share_of_fp64_peak=round(fp64, 3), bound="fp64" if fp64 > hbm else "hbm")
            cases.append(case)
            del t
            work = out = None
    print(json.dumps({"bench": "filters", "device": torch.cuda.get_device_name(0), "power_limit": power_limit(),
                      "hbm_peak_datasheet_tb_s": 3.35, "fp64_peak_datasheet_tflop_s": 34,
                      "timing": "CUDA events, mean of %d after a warm-up" % args.iters, "cases": cases}))


if __name__ == "__main__":
    main()
