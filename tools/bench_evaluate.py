"""Benchmark of `evaluate-segmentation` on the GPU (csrc/evaluate.cu): one JSON line.

    python tools/bench_evaluate.py [--sizes 512 1024] [--iters 5]

Cases: cubes of 512^3 and 1024^3 voxels; uint32 and uint64 label pairs; "blobs" (coherent 16 x 32 x 32 blocks, the ground
truth's blocks shifted by half a block in y and x, so that every block meets four ground-truth ids: long runs of equal pairs)
and "salt" (every voxel an independent random id of 1000 per side: no runs, up to 10^6 distinct pairs, the worst case for
run aggregation; a table of every distinct pair of random 64-bit ids would not fit in memory at 1024^3).

Per case: the contingency pass (table + statistics, cfb_contingency_device) and one scoring call (cfb_contingency_scores)
timed with CUDA events after a warm-up, Mvoxels/s, and the algorithmic bytes (each input read once) over the pass time as a
share of the 3.35 TB/s HBM3 peak of the H100 SXM data sheet.  table_bytes is a lower bound of the traffic the hash tables add
(clearing and scanning the slots, each entry's keys and count, its row and column entries), not counting repeated atomics on
the same slot.  The device name and power limit are read in the same run.
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


def make_pair(torch, size, kind, wide):
    z = torch.arange(size, device="cuda", dtype=torch.int64).view(-1, 1, 1)
    y = torch.arange(size, device="cuda", dtype=torch.int64).view(1, -1, 1)
    x = torch.arange(size, device="cuda", dtype=torch.int64).view(1, 1, -1)
    if kind == "blobs":
        seg = (z // 16) * 1_000_003 + (y // 32) * 1009 + (x // 32) + 1
        gt = (z // 16) * 1_000_003 + ((y + 16) // 32) * 1009 + ((x + 16) // 32) + 7
    else:
        g = torch.Generator(device="cuda").manual_seed(0)
        seg = torch.randint(0, 1000, (size, size, size), device="cuda", generator=g, dtype=torch.int64)
        gt = torch.randint(0, 1000, (size, size, size), device="cuda", generator=g, dtype=torch.int64)
    if wide:   # spread the ids over the whole 64-bit range (an odd multiplier is a bijection modulo 2^64)
        seg = seg * -7046029254386353131
        gt = gt * -7046029254386353131
        return seg.contiguous(), gt.contiguous()
    return seg.to(torch.int32).contiguous(), gt.to(torch.int32).contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[512, 1024])
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    import torch
    from chunkflow_b200 import _native
    if not torch.cuda.is_available():
        raise SystemExit("bench_evaluate needs a CUDA device")
    stream = torch.cuda.current_stream().cuda_stream
    cases = []
    for size in args.sizes:
        for wide in (False, True):
            for kind in ("blobs", "salt"):
                seg, gt = make_pair(torch, size, kind, wide)
                code = _native.DTYPE_U64 if wide else _native.DTYPE_U32
                n = seg.numel()
                slots = 1 << 22
                work = torch.empty(_native.evaluate_workspace(slots), dtype=torch.uint8, device="cuda")
                pairs = _native.contingency_device(seg.data_ptr(), code, gt.data_ptr(), code, seg.shape, work.data_ptr(), slots, stream)
                assert 2 * pairs <= slots
                _native.contingency_scores(work.data_ptr(), slots, 1000, stream)   # warm-up of both calls done
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
                pass_ms = score_ms = 0.0
                for _ in range(args.iters):
                    ev[0].record()
                    _native.contingency_device(seg.data_ptr(), code, gt.data_ptr(), code, seg.shape, work.data_ptr(), slots, stream)
                    ev[1].record()
                    st = _native.contingency_scores(work.data_ptr(), slots, 1000, stream)
                    ev[2].record()
                    torch.cuda.synchronize()
                    pass_ms += ev[0].elapsed_time(ev[1]) / args.iters
                    score_ms += ev[1].elapsed_time(ev[2]) / args.iters
                in_bytes = n * 2 * seg.element_size()
                table_bytes = slots * (8 * 4 + 4 + 4 + 4 + 4) + pairs * (8 + 8 + 4 + 2 * (8 + 4 + 4))
                cases.append(dict(size=size, dtype="uint64" if wide else "uint32", kind=kind, voxels=n, pairs=pairs,
                                  table_slots=slots, pass_ms=round(pass_ms, 3), scores_ms=round(score_ms, 3),
                                  mvoxels_per_s=round(n / (pass_ms * 1e-3) / 1e6, 1), input_bytes=in_bytes,
                                  input_gb_per_s=round(in_bytes / (pass_ms * 1e-3) / 1e9, 1),
                                  share_of_hbm_peak=round(in_bytes / (pass_ms * 1e-3) / HBM_PEAK, 3),
                                  table_bytes=table_bytes, rand_index=st.rand_index))
                del seg, gt, work
                torch.cuda.empty_cache()
    print(json.dumps({"bench": "evaluate_segmentation", "device": torch.cuda.get_device_name(0), "power_limit": power_limit(),
                      "hbm_peak_datasheet_tb_s": 3.35, "timing": "CUDA events, mean of %d after a warm-up" % args.iters,
                      "oracle_cpu_256": "not measured", "cases": cases}))


if __name__ == "__main__":
    main()
