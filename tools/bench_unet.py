"""Step time of the 2-, 3- and 4-level U-Nets on the 1024^3 geometry of bench.py (one H100).

    python tools/bench_unet.py [--steps 3] [--warmup 1] [--depths 2 3 4] [--precision f16f8] [--out FILE]

For every depth: a uint8 1024^3 chunk resident on the device, patch 32x256x256, overlap 8x64x64, 12 patches in flight, the
whole-chunk device path (`infer_chunk_device`, as bench.py times it).  Prints one JSON line per depth with the step time,
the per-layer times of one extra profiled step (CUDA events around every launch), the algorithmic FLOP per patch voxel
(`flops_per_voxel` of the model file: 3x3x3 convolutions, transposed convolutions and the head; pools not counted), the
achieved TFLOP/s over the step and its share of the 989 TFLOP/s dense FP16 figure of the H100 SXM data sheet, and the
device name and power limit read in the same run.  Depth 3 is the seeded network of bench.py; depths 2 and 4 are seeded
checkpoints of the same model file.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
MODEL_FILE = os.path.join(ROOT, "chunkflow_b200", "convnet", "unet3l.py")
CHUNK, PATCH, OVERLAP = (1024, 1024, 1024), (32, 256, 256), (8, 64, 64)
PEAK_TFLOPS = 989.0  # H100 SXM data sheet, dense FP16 / BF16, 700 W


def device_info(index):
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                        "-i", str(index)], capture_output=True, text=True)
    name, power, clock = (s.strip() for s in q.stdout.strip().split(","))
    return {"device": name, "power_limit_w": float(power), "max_sm_clock_mhz": float(clock)}


def run_depth(depth, weights, args, d_in, model_src):
    import torch
    from chunkflow_b200 import Inferencer
    inf = Inferencer(MODEL_FILE, weights, PATCH, output_patch_overlap=OVERLAP, num_output_channels=3, framework="b200",
                     batch_size=args.batch_size, mask_output_chunk=True, precision=args.precision)
    eng = inf.engine
    d_out = torch.empty(eng.output_shape(CHUNK), dtype=torch.float32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream

    def step():
        eng.infer_chunk_device(d_in.data_ptr(), np.uint8, CHUNK, d_out.data_ptr(), stream)

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    launches = eng.last_timing()["launches"]
    eng.set_profiling(True)
    step()
    torch.cuda.synchronize()
    layers = {k: round(v[0], 3) for k, v in eng.layer_timing().items()}
    eng.set_profiling(False)
    patches = len(eng.patch_grid(CHUNK))
    flop_per_voxel = model_src.flops_per_voxel(depth, 3)
    flop = flop_per_voxel * patches * int(np.prod(PATCH))
    tflops = flop / (ms / 1e3) / 1e12
    finite = bool(torch.isfinite(d_out).all().item())
    eng.close()
    del d_out, inf
    torch.cuda.empty_cache()
    return {"depth": depth, "widths": list(model_src.widths(depth)), "precision": args.precision or "f16f8",
            "ms_per_step": round(ms, 2), "launches_per_step": launches, "patches_per_step": patches,
            "flop_per_patch_voxel": flop_per_voxel, "tflops": round(tflops, 1),
            "share_of_989_tflops": round(tflops / PEAK_TFLOPS, 4), "layer_ms": layers, "output_finite": finite}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--depths", type=int, nargs="+", default=[2, 3, 4])
    ap.add_argument("--batch-size", type=int, default=12)
    ap.add_argument("--precision", default=None, help="simt, f16x3, f16f8 (default) or f16")
    ap.add_argument("--out", help="also write the JSON lines to this file")
    args = ap.parse_args()

    import torch
    from chunkflow_b200.lib import load_source
    if not torch.cuda.is_available():
        raise SystemExit("bench_unet.py measures on a GPU; none is visible")
    model_src = load_source(MODEL_FILE)
    info = device_info(torch.cuda.current_device())
    g = torch.Generator(device="cuda").manual_seed(20260922)
    d_in = torch.randint(1, 256, CHUNK, dtype=torch.uint8, device="cuda", generator=g)
    lines = []
    with tempfile.TemporaryDirectory() as tmp:
        for depth in args.depths:
            weights = None
            if depth != 3:  # depth 3: the seeded network bench.py times
                weights = os.path.join(tmp, f"unet{depth}.pt")
                torch.save(model_src.create_model(cout=3, depth=depth).state_dict(), weights)
            r = {**run_depth(depth, weights, args, d_in, model_src), **info}
            lines.append(json.dumps(r))
            print(lines[-1], flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
