"""Benchmark of the segmentation clean-up on the GPU (csrc/relabel.cu): one JSON line.

    python tools/bench_relabel.py [--sizes 512 1024] [--iters 5]

Cases: cubes of 512^3 and 1024^3 voxels; uint32 and uint64 labels; "blobs" (coherent 16 x 32 x 32 blocks of one id each: long
runs) and "salt" (every voxel an independent random id of 10^6: no runs, the worst case for run aggregation).

Per case, timed with CUDA events after a warm-up: the count pass (cfb_label_table_device), the plan (cfb_label_table_plan) and
the apply pass (cfb_label_apply_device) of `mask-out-objects -d T -s ids` (output of the input's width) and of `remap` (uint64
output), and both operations end to end through DeviceChunk (table sizing and allocation included).  Algorithmic bytes -- count:
the volume read once; apply: the volume read once and the output written once -- over the pass time, as a share of the
3.35 TB/s HBM3 peak of the H100 SXM data sheet (a data-sheet figure, not a measured one).  The device name and power limit are
read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

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


def make_labels(torch, size, kind, wide):
    if kind == "blobs":
        z = torch.arange(size, device="cuda", dtype=torch.int64).view(-1, 1, 1)
        y = torch.arange(size, device="cuda", dtype=torch.int64).view(1, -1, 1)
        x = torch.arange(size, device="cuda", dtype=torch.int64).view(1, 1, -1)
        seg = ((z // 16) * 1_000_003 + (y // 32) * 1009 + (x // 32)).expand(size, size, size)
    else:
        g = torch.Generator(device="cuda").manual_seed(0)
        seg = torch.randint(0, 1_000_000, (size, size, size), device="cuda", generator=g, dtype=torch.int64)
    if wide:   # spread the ids over the whole 64-bit range (an odd multiplier is a bijection modulo 2^64)
        return (seg * -7046029254386353131).contiguous()
    return seg.to(torch.int32).contiguous()


def timed(torch, iters, fn):
    fn()
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
        raise SystemExit("bench_relabel needs a CUDA device")
    stream = torch.cuda.current_stream().cuda_stream
    share = lambda nbytes, ms: round(nbytes / (ms * 1e-3) / HBM_PEAK, 3)
    cases = []
    for size in args.sizes:
        for wide in (False, True):
            for kind in ("blobs", "salt"):
                seg = make_labels(torch, size, kind, wide)
                code = _native.DTYPE_U64 if wide else _native.DTYPE_U32
                n, width = seg.numel(), seg.element_size()
                slots = 1 << 22
                work = torch.empty(_native.label_table_workspace(n, slots), dtype=torch.uint8, device="cuda")
                num = _native.label_table_device(seg.data_ptr(), code, seg.shape, work.data_ptr(), slots, stream)
                assert 2 * num <= slots
                ids, counts, _ = _native.label_table_read(work.data_ptr(), slots, num, stream)
                thr = int(np.median(counts))
                keep = torch.from_numpy(ids[::2].copy().view(np.int64)).cuda()
                same = torch.empty_like(seg)
                out64 = torch.empty(seg.shape, dtype=torch.int64, device="cuda")
                count_ms = timed(torch, args.iters, lambda: _native.label_table_device(seg.data_ptr(), code, seg.shape, work.data_ptr(),
                                                                                      slots, stream))
                plan_mask_ms = timed(torch, args.iters, lambda: _native.label_table_plan(work.data_ptr(), slots, n, thr, keep.data_ptr(),
                                                                                        keep.numel(), False, 0, stream))
                apply_mask_ms = timed(torch, args.iters, lambda: _native.label_apply_device(seg.data_ptr(), code, n, work.data_ptr(), slots,
                                                                                          same.data_ptr(), code, stream))
                plan_remap_ms = timed(torch, args.iters, lambda: _native.label_table_plan(work.data_ptr(), slots, n, None, 0, None, True, 0,
                                                                                         stream))
                apply_remap_ms = timed(torch, args.iters, lambda: _native.label_apply_device(seg.data_ptr(), code, n, work.data_ptr(), slots,
                                                                                           out64.data_ptr(), _native.DTYPE_U64, stream))
                survivors = _native.label_table_plan(work.data_ptr(), slots, n, None, 0, None, True, 0, stream)[1]
                del work, same, out64

                def mask_e2e():
                    DeviceChunk(seg.clone()).mask_out_objects(thr, ids[::2])

                def remap_e2e():
                    DeviceChunk(seg.clone()).remap()

                clone_ms = timed(torch, args.iters, lambda: seg.clone())
                mask_ms = timed(torch, args.iters, mask_e2e) - clone_ms
                remap_ms = timed(torch, args.iters, remap_e2e) - clone_ms
                cases.append(dict(size=size, dtype="uint64" if wide else "uint32", kind=kind, voxels=n, labels=num,
                                  survivors_of_remap=survivors, table_slots=slots, dust_threshold=thr, keep_ids=int(keep.numel()),
                                  count_ms=round(count_ms, 3), count_share_of_hbm_peak=share(n * width, count_ms),
                                  plan_mask_ms=round(plan_mask_ms, 3), apply_mask_ms=round(apply_mask_ms, 3),
                                  apply_mask_share_of_hbm_peak=share(2 * n * width, apply_mask_ms),
                                  plan_remap_ms=round(plan_remap_ms, 3), apply_remap_ms=round(apply_remap_ms, 3),
                                  apply_remap_share_of_hbm_peak=share(n * (width + 8), apply_remap_ms),
                                  mask_out_objects_ms=round(mask_ms, 3), remap_ms=round(remap_ms, 3)))
                del seg, keep
                torch.cuda.empty_cache()
    print(json.dumps({"bench": "relabel", "device": torch.cuda.get_device_name(0), "power_limit": power_limit(),
                      "hbm_peak_datasheet_tb_s": 3.35,
                      "timing": "CUDA events, mean of %d after a warm-up; end-to-end times exclude the clone of the input" % args.iters,
                      "cases": cases}))


if __name__ == "__main__":
    main()
