"""``chunkflow``-style command line for the inference hot path.

Chained multi-command group with lazily pulled operator generators, like the reference
(chunkflow/lib/flow.py:44-105).  The two commands on the hot path, plus the operators either side of it on the GPU
(`normalize-contrast`, `crop-margin`, `quantize`; `to-device` / `to-host` keep the chunk in GPU memory in between):

    python -m chunkflow_b200.flow.cli create-chunk --size 64 256 256 \
        inference --input-patch-size 20 256 256 --output-patch-overlap 4 64 64 \
                  --num-output-channels 3 --framework b200 --batch-size 12 --mask-output-chunk

``inference`` keeps every flag of the reference operator (chunkflow/flow/flow.py:1853-1893) and adds
the ``b200`` framework choice; ``-f pytorch`` is accepted for the canonical model file.
"""
from functools import update_wrapper
from time import time

import click
import numpy as np

from chunkflow_b200.chunk import Chunk

state = {"dry_run": False, "verbose": 1}


def default_none(ctx, _, value):
    """click turns a missing nargs=3 option into an empty tuple; the operators expect None."""
    return None if value is None or len(value) == 0 else value


@click.group(chain=True)
@click.option("--mip", type=click.INT, default=0, help="default mip level of chunks.")
@click.option("--dry-run/--real-run", default=False, help="dry run or real run.")
@click.option("--verbose/--quiet", default=True, help="print informations or not.")
def main(mip, dry_run, verbose):
    """Compose operators and create your own pipeline (inference hot path only)."""
    state["mip"] = mip
    state["dry_run"] = dry_run
    state["verbose"] = verbose


@main.result_callback()
def process_commands(operators, mip, dry_run, verbose):
    stream = [{"log": {"timer": {}}}]
    for op in operators:
        stream = op(stream)
    tasks = []
    for task in stream:   # pull-driven execution
        tasks.append(task)
    return tasks


def operator(func):
    """Wrap a command so that it returns a closure over the task stream (reference lib/flow.py:82-93)."""
    def new_func(*args, **kwargs):
        def op(stream):
            return func(stream, *args, **kwargs)
        return op
    return update_wrapper(new_func, func)


@main.command("create-chunk")
@click.option("--name", type=str, default="create-chunk", help="name of operator")
@click.option("--size", "-s", type=click.INT, nargs=3, default=(64, 64, 64), help="the size of created chunk")
@click.option("--dtype", "-d", type=click.Choice(["uint8", "float32", "float64"]), default="uint8",
              help="the data type of chunk (the reference's integer label types need cc3d and are not part of this path)")
@click.option("--pattern", "-p", type=click.Choice(["sin", "random", "zero"]), default="sin")
@click.option("--voxel-offset", "-t", type=click.INT, nargs=3, default=(0, 0, 0), help="offset in voxel number.")
@click.option("--voxel-size", "-e", type=click.INT, nargs=3, default=(1, 1, 1), help="voxel size in nm")
@click.option("--output-chunk-name", "-o", type=str, default="chunk", help="name of created chunk")
@operator
def create_chunk(tasks, name, size, dtype, pattern, voxel_offset, voxel_size, output_chunk_name):
    """Create a fake chunk for easy test (reference flow/flow.py:652-678)."""
    for task in tasks:
        task[output_chunk_name] = Chunk.create(size=size, dtype=np.dtype(dtype), pattern=pattern,
                                               voxel_offset=voxel_offset, voxel_size=voxel_size)
        yield task


@main.command("inference")
@click.option("--name", type=str, default="inference", help="name of this operator")
@click.option("--convnet-model", "-m", type=str, default=None, help="convnet model path or type.")
@click.option("--convnet-weight-path", "-w", type=str, default=None, help="convnet weight path")
@click.option("--input-patch-size", "-s", type=click.INT, nargs=3, required=True, help="input patch size")
@click.option("--output-patch-size", "-z", type=click.INT, nargs=3, default=None, callback=default_none,
              help="output patch size")
@click.option("--output-patch-overlap", "-v", type=click.INT, nargs=3, default=(4, 64, 64), help="patch overlap")
@click.option("--output-crop-margin", type=click.INT, nargs=3, default=None, callback=default_none,
              help="margin size of output chunk cropping.")
@click.option("--patch-num", "-n", default=None, callback=default_none, type=click.INT, nargs=3,
              help="patch number in z,y,x.")
@click.option("--num-input-channels", type=click.INT, default=1, help="number of input channels")
@click.option("--num-output-channels", "-c", type=click.INT, default=3, help="number of output channels")
@click.option("--dtype", "-d", type=click.Choice(["float32", "float16"]), default="float32",
              help="float32: fp16 hi/lo split tensor-core arithmetic with fp32 accumulation (1e-3 parity mode); "
                   "float16: single-pass fp16 tensor cores. The result is float32 either way.")
@click.option("--framework", "-f", type=click.Choice(["universal", "identity", "pytorch", "b200"]), default="universal",
              help="inference framework")
@click.option("--batch-size", "-b", type=click.INT, default=1, help="mini batch size of input patch.")
@click.option("--bump", type=click.Choice(["wu", "zung"]), default="wu", help="bump function type (only support wu now!).")
@click.option("--mask-output-chunk/--no-mask-output-chunk", default=False,
              help="mask output chunk will make the whole chunk like one output patch. "
                   "This will also work with non-aligned chunk size.")
@click.option("--mask-myelin-threshold", "-y", default=None, type=click.FLOAT,
              help="mask myelin if netoutput have myelin channel.")
@click.option("--augment/--no-augment", default=False,
              help="transform the input patch and transform back the output patch")
@click.option("--input-chunk-name", "-i", type=str, default="chunk", help="input chunk name")
@click.option("--output-chunk-name", "-o", type=str, default="chunk", help="output chunk name")
@operator
def inference(tasks, name, convnet_model, convnet_weight_path, input_patch_size, output_patch_size,
              output_patch_overlap, output_crop_margin, patch_num, num_input_channels, num_output_channels, dtype,
              framework, batch_size, bump, mask_output_chunk, mask_myelin_threshold, augment, input_chunk_name,
              output_chunk_name):
    """Perform convolutional network inference for chunks (reference flow/flow.py:1894-1933)."""
    from chunkflow_b200.flow.divid_conquer.inferencer import Inferencer
    with Inferencer(
            convnet_model, convnet_weight_path,
            input_patch_size=input_patch_size, output_patch_size=output_patch_size,
            num_input_channels=num_input_channels, num_output_channels=num_output_channels,
            output_patch_overlap=output_patch_overlap, output_crop_margin=output_crop_margin,
            patch_num=patch_num, framework=framework, dtype=dtype, batch_size=batch_size, bump=bump,
            augment=augment, mask_output_chunk=mask_output_chunk, mask_myelin_threshold=mask_myelin_threshold,
            dry_run=state["dry_run"]) as inferencer:
        for task in tasks:
            if task is not None:
                if "log" not in task:
                    task["log"] = {"timer": {}}
                start = time()
                chunk_in = task[input_chunk_name]
                if isinstance(chunk_in, Chunk) or inferencer.patch_inferencer is not None or state["dry_run"]:
                    task[output_chunk_name] = inferencer(_to_host(chunk_in))
                else:  # a DeviceChunk (see `to-device`): the result stays in GPU memory too
                    task[output_chunk_name] = inferencer.infer_device(chunk_in)
                task["log"]["timer"][name] = time() - start
                task["log"]["compute_device"] = inferencer.compute_device
                if state["verbose"]:
                    out = task[output_chunk_name]
                    print(f"{name}: {out.shape} in {task['log']['timer'][name]:.3f} s on "
                          f"{task['log']['compute_device']} ({np.prod(out.shape[-3:]) / task['log']['timer'][name] / 1e6:.1f} Mvoxels/s)")
            yield task


# ---------------------------------------------------------------------------------------------
# operators either side of `inference`, on the GPU (SURVEY.md section 8 f3).  A task's chunk is either a host
# `Chunk` (moved to the GPU for the kernel and back, like `inference` does) or -- after `to-device` -- a `DeviceChunk`
# that stays in GPU memory from operator to operator until `to-host`.
# ---------------------------------------------------------------------------------------------
def _to_host(chunk):
    return chunk if isinstance(chunk, Chunk) else chunk.to_chunk()


def _on_device(chunk, device):
    """(DeviceChunk, was_host)"""
    from chunkflow_b200.chunk.device import DeviceChunk
    if isinstance(chunk, DeviceChunk):
        return chunk, False
    return DeviceChunk.from_chunk(chunk, device=device), True


@main.command("to-device")
@click.option("--device", type=str, default="cuda:0", help="GPU that will hold the chunk between operators.")
@click.option("--input-chunk-name", "-i", type=str, default="chunk", help="input chunk name")
@click.option("--output-chunk-name", "-o", type=str, default="chunk", help="output chunk name")
@operator
def to_device(tasks, device, input_chunk_name, output_chunk_name):
    """(extension) Move the chunk to GPU memory; the following operators run on it there."""
    for task in tasks:
        if task is not None:
            task[output_chunk_name] = _on_device(task[input_chunk_name], device)[0]
        yield task


@main.command("to-host")
@click.option("--input-chunk-name", "-i", type=str, default="chunk", help="input chunk name")
@click.option("--output-chunk-name", "-o", type=str, default="chunk", help="output chunk name")
@operator
def to_host(tasks, input_chunk_name, output_chunk_name):
    """(extension) Bring a GPU-resident chunk back to host memory."""
    for task in tasks:
        if task is not None:
            task[output_chunk_name] = _to_host(task[input_chunk_name])
        yield task


@main.command("normalize-contrast")
@click.option("--name", type=str, default="normalize-contrast-nkem", help="name of operator.")
@click.option("--input-chunk-name", "-i", type=str, default="chunk", help="input chunk name")
@click.option("--output-chunk-name", "-o", type=str, default="chunk", help="output chunk name")
@click.option("--lower-clip-fraction", "-l", type=click.FLOAT, default=0.01, help="lower intensity fraction to clip out.")
@click.option("--upper-clip-fraction", "-u", type=click.FLOAT, default=0.01, help="upper intensity fraction to clip out.")
@click.option("--minval", type=click.INT, default=1, help="the minimum intensity of transformed chunk.")
@click.option("--maxval", type=click.INT, default=255, help="the maximum intensity of transformed chunk.")
@click.option("--per-section/--whole", default=True, help="per section normalization or normalize the whole chunk.")
@operator
def normalize_contrast(tasks, name, input_chunk_name, output_chunk_name, lower_clip_fraction, upper_clip_fraction, minval,
                       maxval, per_section):
    """Normalize the section contrast (reference flow/flow.py:1672-1711, chunk/image/base.py:93-132)."""
    import torch
    from chunkflow_b200.chunk.device import DeviceChunk
    for task in tasks:
        if task is not None:
            start = time()
            dev, was_host = _on_device(task[input_chunk_name], "cuda:0")
            if not was_host:  # the reference works on a clone (flow.py:1699)
                dev = DeviceChunk(dev.tensor.clone(), voxel_offset=dev.voxel_offset, voxel_size=dev.voxel_size)
            dev.normalize_contrast(lower_clip_fraction=lower_clip_fraction, upper_clip_fraction=upper_clip_fraction,
                                   minval=minval, maxval=maxval, per_section=per_section)
            torch.cuda.synchronize(dev.tensor.device)
            task[output_chunk_name] = dev.to_chunk() if was_host else dev
            task["log"]["timer"][name] = time() - start
        yield task


@main.command("crop-margin")
@click.option("--name", type=str, default="crop-margin", help="name of this operator")
@click.option("--margin-size", "-m", type=click.INT, nargs=6, default=None, callback=default_none,
              help="crop the chunk margin: -z -y -x +z +y +x.")
@click.option("--input-chunk-name", "-i", type=str, default="chunk", help="input chunk name.")
@click.option("--output-chunk-name", "-o", type=str, default="chunk", help="output chunk name.")
@operator
def crop_margin(tasks, name, margin_size, input_chunk_name, output_chunk_name):
    """Crop the margin of chunk (reference flow/flow.py:2053-2084; the bounding-box form needs a task bbox and is not
    part of this path)."""
    import torch
    if not margin_size:
        raise click.UsageError("crop-margin: --margin-size is required here (no task bounding boxes on this path)")
    for task in tasks:
        if task is not None:
            start = time()
            dev, was_host = _on_device(task[input_chunk_name], "cuda:0")
            out = dev.crop_margin(margin_size)
            torch.cuda.synchronize(out.tensor.device)
            task[output_chunk_name] = out.to_chunk() if was_host else out
            task["log"]["timer"][name] = time() - start
        yield task


@main.command("quantize")
@click.option("--input-chunk-name", "-i", type=str, default="chunk", help="input chunk name")
@click.option("--output-chunk-name", "-o", type=str, default="chunk", help="output chunk name")
@click.option("--mode", type=click.Choice(["xy", "z"]), default="xy", help="xy: average of xy channel; z: only the z channel")
@operator
def quantize(tasks, input_chunk_name, output_chunk_name, mode):
    """Transform an affinity map to a uint8 image (reference flow/flow.py:2250-2273, chunk/affinity_map/base.py:33-57)."""
    import torch
    for task in tasks:
        if task is not None:
            dev, was_host = _on_device(task[input_chunk_name], "cuda:0")
            out = dev.quantize(mode=mode)
            torch.cuda.synchronize(out.tensor.device)
            task[output_chunk_name] = out.to_chunk() if was_host else out
        yield task


@main.command("connected-components")
@click.option("--name", type=str, default="connected-components", help="threshold a map and get the targets.")
@click.option("--input-chunk-name", "-i", type=str, default="chunk", help="input chunk name")
@click.option("--output-chunk-name", "-o", type=str, default="chunk", help="output chunk name")
@click.option("--threshold", "-t", type=click.FLOAT, default=None, help="threshold to cut the map.")
@click.option("--connectivity", "-c", type=click.Choice(["6", "18", "26"]), default="6",
              help="number of neighboring voxels used. Default is 6.")
@operator
def connected_components(tasks, name, input_chunk_name, output_chunk_name, threshold, connectivity):
    """Threshold the probability map to get a segmentation (reference flow/flow.py:1803-1830, chunk/base.py:128-137)."""
    import torch
    connectivity = int(connectivity)
    for task in tasks:
        if task is not None:
            start = time()
            dev, was_host = _on_device(task[input_chunk_name], "cuda:0")
            out = dev.connected_component(threshold=threshold, connectivity=connectivity)
            torch.cuda.synchronize(out.tensor.device)
            task[output_chunk_name] = out.to_chunk() if was_host else out
            task["log"]["timer"][name] = time() - start
        yield task


@main.command("agglomerate")
@click.option("--name", type=str, default="agglomerate", help="name of this operator")
@click.option("--input-chunk-name", "-i", type=str, default="chunk", help="input chunk name (the affinity map)")
@click.option("--output-chunk-name", "-o", type=str, default="chunk", help="output chunk name (the segmentation)")
@click.option("--threshold", "-t", type=click.FLOAT, default=0.7, help="merge until the score (1 - mean affinity by default) reaches this.")
@click.option("--aff-threshold-low", type=click.FLOAT, default=0.001, help="watershed: affinities up to this are no edges.")
@click.option("--aff-threshold-high", type=click.FLOAT, default=0.9999, help="watershed: affinities from this on always connect.")
@click.option("--flip-channel/--no-flip-channel", default=True,
              help="the channels are stored x, y, z (chunkflow) and read in reverse (waterz wants z, y, x).")
@click.option("--scoring-function", type=str, default='OneMinus<MeanAffinity<RegionGraphType, ScoreValue>>',
              help="waterz's scoring function: the mean affinity, or "
                   "'OneMinus<HistogramQuantileAffinity<RegionGraphType, Q, ScoreValue, B[, I]>>'.")
@operator
def agglomerate(tasks, name, input_chunk_name, output_chunk_name, threshold, aff_threshold_low, aff_threshold_high, flip_channel,
                scoring_function):
    """Watershed + agglomeration of an affinity map (the reference runs this as `plugin -f agglomerate`:
    plugins/agglomerate.py:8-48 -> waterz.agglomerate; README.md:39)."""
    from chunkflow_b200.chunk.device import parse_scoring_function
    parse_scoring_function(scoring_function)
    import torch
    for task in tasks:
        if task is not None:
            start = time()
            dev, was_host = _on_device(task[input_chunk_name], "cuda:0")
            out = dev.agglomerate(threshold=threshold, aff_threshold_low=aff_threshold_low, aff_threshold_high=aff_threshold_high,
                                  flip_channel=flip_channel, scoring_function=scoring_function)
            torch.cuda.synchronize(out.tensor.device)
            task[output_chunk_name] = out.to_chunk() if was_host else out
            task["log"]["timer"][name] = time() - start
        yield task


@main.command("downsample")
@click.option("--input-chunk-name", "-i", type=str, default="chunk", help="input chunk name")
@click.option("--output-chunk-name", "-o", type=str, default="chunk", help="output chunk name")
@click.option("--factor", "-f", type=click.INT, nargs=3, default=(2, 2, 2), help="downsample factor in zyx. The default is 2x2x2.")
@operator
def downsample(tasks, input_chunk_name, output_chunk_name, factor):
    """Downsample a chunk (reference flow/flow.py:1545-1573): a uint8 image is averaged, an integer or boolean segmentation
    mode-pooled.  A pyramid is a chain (`downsample -o mip1 downsample -i mip1 -o mip2`), a thumbnail
    `quantize --mode z downsample -f 1 2 2 ...`.  A host chunk comes back to the host, a GPU-resident one stays there."""
    import torch
    for task in tasks:
        if task is not None:
            dev, was_host = _on_device(task[input_chunk_name], "cuda:0")
            out = dev.downsample(factor)
            torch.cuda.synchronize(out.tensor.device)
            if was_host:
                out = Chunk(out.to_chunk().array, voxel_offset=out.voxel_offset, voxel_size=out.voxel_size,
                            layer_type=getattr(task[input_chunk_name], "_layer_type", None))
            task[output_chunk_name] = out
        yield task


@main.command("gaussian-filter")
@click.option("--name", type=str, default="gaussian-filter", help="name of operator")
@click.option("--input-chunk-name", "-i", type=str, default="chunk", help="input chunk name")
@click.option("--sigma", "-s", type=click.INT, default=1, help="standard deviation of gaussian kernel")
@operator
def gaussian_filter(tasks, name, input_chunk_name, sigma):
    """2D Gaussian blurring operated in-place (reference flow/flow.py:1615-1630), bit-identical to scipy.ndimage.  On a
    (c,z,y,x) chunk the blur also runs across the channels, as in the reference.  A host chunk's array is written in place,
    a GPU-resident chunk is filtered where it is."""
    import torch
    for task in tasks:
        if task is not None:
            start = time()
            chunk = task[input_chunk_name]
            chunk.gaussian_filter_2d(sigma)
            if not isinstance(chunk, Chunk):
                torch.cuda.synchronize(chunk.tensor.device)
            task["log"]["timer"][name] = time() - start
        yield task


@main.command("median-filter")
@click.option("--input-chunk-name", "-i", type=str, default="chunk", help="input chunk name")
@click.option("--output-chunk-name", "-o", type=str, default="chunk", help="output chunk name")
@click.option("--size", "-s", type=click.INT, nargs=3, default=(3, 1, 1), help="window size in zyx. The default is 3x1x1.")
@click.option("--mode", type=click.Choice(["reflect", "nearest", "mirror", "wrap", "constant", "grid-mirror", "grid-wrap",
                                           "grid-constant"]), default="reflect", help="boundary mode (constant: 0)")
@operator
def median_filter(tasks, input_chunk_name, output_chunk_name, size, mode):
    """(extension) Median filter, bit-identical to scipy.ndimage.median_filter: the reference runs it as
    `plugin -f median_filter` (plugins/median_filter.py).  The default 3x1x1 suppresses a single bad section across z.
    A host chunk comes back to the host, a GPU-resident one stays there."""
    import torch
    for task in tasks:
        if task is not None:
            dev, was_host = _on_device(task[input_chunk_name], "cuda:0")
            out = dev.median_filter(size, mode)
            torch.cuda.synchronize(out.tensor.device)
            if was_host:
                out = Chunk(out.to_chunk().array, voxel_offset=out.voxel_offset, voxel_size=out.voxel_size,
                            layer_type=getattr(task[input_chunk_name], "_layer_type", None))
            task[output_chunk_name] = out
        yield task


@main.command("clahe")
@click.option("--input-chunk-name", "-i", type=str, default="chunk", help="input chunk name")
@click.option("--output-chunk-name", "-o", type=str, default="chunk", help="output chunk name")
@click.option("--clip-limit", "-c", type=click.FLOAT, default=20.0, help="contrast limit; 0 or less: no clipping.")
@click.option("--tile-grid-size", "-t", type=click.INT, nargs=2, default=(512, 512),
              help="number of tiles in x and y (OpenCV's order, x first).")
@operator
def clahe(tasks, input_chunk_name, output_chunk_name, clip_limit, tile_grid_size):
    """(extension) Contrast-limited adaptive histogram equalization of every z section of a uint8 image, bit-identical to
    cv2.createCLAHE(clip_limit, tile_grid_size).apply: the reference runs it as `plugin -f clahe` (plugins/clahe.py).
    A host chunk comes back to the host, a GPU-resident one stays there."""
    import torch
    for task in tasks:
        if task is not None:
            dev, was_host = _on_device(task[input_chunk_name], "cuda:0")
            out = dev.clahe(clip_limit, tile_grid_size)
            torch.cuda.synchronize(out.tensor.device)
            if was_host:
                out = Chunk(out.to_chunk().array, voxel_offset=out.voxel_offset, voxel_size=out.voxel_size,
                            layer_type=getattr(task[input_chunk_name], "_layer_type", None))
            task[output_chunk_name] = out
        yield task


@main.command("evaluate-segmentation")
@click.option("--segmentation-chunk-name", "-s", type=str, default="chunk", help="chunk name of segmentation")
@click.option("--groundtruth-chunk-name", "-g", type=str, default="groundtruth")
@click.option("--output", "-o", type=str, default="seg_score", help="segmentation evaluation result name.")
@operator
def evaluate_segmentation(tasks, segmentation_chunk_name, groundtruth_chunk_name, output):
    """Evaluate segmentation by split/merge error (reference flow/flow.py:1519-1542, chunk/segmentation.py:33-67).  The
    chunks may be host chunks (uploaded for the call) or GPU-resident ones."""
    from chunkflow_b200.chunk.segmentation import evaluate
    for task in tasks:
        if task is not None:
            task[output] = evaluate(task[segmentation_chunk_name], task[groundtruth_chunk_name])
        yield task


@main.command("mask-out-objects")
@click.option("--input-chunk-name", "-i", type=str, default="chunk")
@click.option("--output_chunk_name", "-o", type=str, default="chunk")
@click.option("--dust-size-threshold", "-d", type=click.INT, default=None,
              help="eliminate small objects with voxel number less than or equal to threshold.")
@click.option("--selected-obj-ids", "-s", type=str, default=None,
              help="a list of segment ids to keep. This is for sparse meshing. The ids should be separated by comma without "
                   "space, such as \"34,56,78,90\"; it can also be a local json file that contains a list of ids.")
@operator
def mask_out_objects(tasks, input_chunk_name, output_chunk_name, dust_size_threshold, selected_obj_ids):
    """Mask out objects in a segmentation chunk (reference flow/flow.py:2015-2050): dust first, then everything outside the
    selection, in one pass over the table of labels and one over the volume.  A host chunk gives a host Segmentation, a
    GPU-resident chunk is changed where it is."""
    from chunkflow_b200.chunk.device import DeviceChunk, selected_ids
    from chunkflow_b200.chunk.segmentation import Segmentation, mask_out_objects as run
    if selected_obj_ids is not None:
        selected_obj_ids = selected_ids(selected_obj_ids)   # parsed (and a json file read) once, like the reference
    for task in tasks:
        if task is not None:
            seg = task[input_chunk_name]
            if not isinstance(seg, (Segmentation, DeviceChunk)):
                assert isinstance(seg, Chunk)
                seg = Segmentation.from_chunk(seg)
            task[output_chunk_name] = run(seg, dust_size_threshold, selected_obj_ids)
        yield task


@main.command("remap-segmentation")
@click.option("--input-chunk-name", "-i", type=str, default="chunk", help="input chunk name")
@click.option("--output-chunk-name", "-o", type=str, default="chunk", help="output chunk name")
@click.option("--base-id", type=click.INT, default=None,
              help="the ids start after this one (default: the task's base_id, the largest id of the previous remap, or 0).")
@operator
def remap_segmentation(tasks, input_chunk_name, output_chunk_name, base_id):
    """(extension) Renumber the object ids to 1..N in raster order of their first voxel, after --base-id (reference
    chunk/segmentation.py:69-84; the reference has the method but no command).  The largest new id is stored in
    task['base_id'], where the next remap of the same invocation starts, so that its chunks get disjoint id ranges."""
    from chunkflow_b200.chunk.device import DeviceChunk
    from chunkflow_b200.chunk.segmentation import Segmentation
    for task in tasks:
        if task is not None:
            seg = task[input_chunk_name]
            if not isinstance(seg, (Segmentation, DeviceChunk)):
                assert isinstance(seg, Chunk)
                seg = Segmentation.from_chunk(seg)
            task["base_id"] = int(seg.remap(task.get("base_id", 0) if base_id is None else base_id))
            task[output_chunk_name] = seg
        yield task


@main.command("fill-segmentation-holes")
@click.option("--input-chunk-name", "-i", type=str, default="chunk", help="input chunk name")
@click.option("--output-chunk-name", "-o", type=str, default="chunk", help="output chunk name")
@click.option("--mode", type=click.Choice(["binary", "keep-enclosed", "remove-enclosed"]), default="binary",
              help="binary: fill_voids.fill (1 for the foreground and its holes); keep-enclosed: every 0 voxel enclosed by an object "
                   "takes the id of the innermost one; remove-enclosed: every enclosed voxel takes the id of the outermost encloser.")
@operator
def fill_segmentation_holes(tasks, input_chunk_name, output_chunk_name, mode):
    """(extension) Fill the holes of a segmentation chunk on the GPU, 6-connected, outside being beyond the chunk's faces
    (the reference runs it as `plugin -f fill_segmentation_holes`, plugins/fill_segmentation_holes.py -> fill_voids.fill; rules
    restated in oracle/fill_holes_oracle.py).  A host chunk comes back to the host, a GPU-resident one stays there."""
    import torch
    for task in tasks:
        if task is not None:
            dev, was_host = _on_device(task[input_chunk_name], "cuda:0")
            out = dev.fill_holes(mode)
            torch.cuda.synchronize(out.tensor.device)
            if was_host:
                out = Chunk(out.to_chunk().array, voxel_offset=out.voxel_offset, voxel_size=out.voxel_size,
                            layer_type=getattr(task[input_chunk_name], "_layer_type", None))
            task[output_chunk_name] = out
        yield task


@main.command("mesh")
@click.option("--name", type=str, default="mesh", help="name of operator")
@click.option("--input-chunk-name", "-i", type=str, default="chunk", help="name of chunk needs to be meshed.")
@click.option("--mip", "-m", type=click.INT, default=None, help="mip level of segmentation chunk.")
@click.option("--voxel-size", "-v", type=click.INT, nargs=3, default=None, callback=default_none,
              help="voxel size of the segmentation. zyx order.")
@click.option("--output-path", "-o", type=str, default="file:///tmp/mesh/",
              help="output path of meshes: a local directory or file:// URL. With the precomputed format, the mesh directory "
                   "named in its info file.")
@click.option("--output-format", "-t", type=click.Choice(["ply", "obj", "precomputed"]), default="precomputed",
              help="output format, could be one of ply|obj|precomputed.")
@click.option("--simplification-factor", "-f", type=click.INT, default=100, help="mesh simplification factor.")
@click.option("--max-simplification-error", "-e", type=click.INT, default=40, help="max simplification error.")
@click.option("--skip-ids", "-s", type=str, default=None, help="do not mesh for some specific ids.")
@click.option("--manifest/--no-manifest", default=False, help="create manifest file or not.")
@click.option("--shard/--no-shard", default=False, help="combine meshes as one file")
@operator
def mesh(tasks, name, input_chunk_name, mip, voxel_size, output_path, output_format, simplification_factor,
         max_simplification_error, skip_ids, manifest, shard):
    """Perform meshing for segmentation chunk (reference flow/flow.py:2087-2135, flow/mesh.py): marching cubes on the GPU,
    welding and simplification on the host (rules restated: not zmesh's meshes).  A host chunk is uploaded for the call, a
    GPU-resident one is meshed where it is."""
    from chunkflow_b200.flow.mesh import MeshWriter
    if mip is None:
        mip = state["mip"]
    if skip_ids is not None:
        skip_ids = frozenset(map(int, skip_ids.split(",")))
    writer = MeshWriter(output_path, output_format, mip=mip, voxel_size=voxel_size, max_simplification_error=max_simplification_error,
                        manifest=manifest, shard=shard)
    for task in tasks:
        if task is not None:
            start = time()
            seg = task[input_chunk_name]
            dev, _ = _on_device(seg, "cuda:0")
            vs = writer.voxel_size if writer.voxel_size is not None else seg.voxel_size
            # the shard holds every object (as in the reference); the fragments skip the ids when they are written
            meshes = dev.mesh(voxel_size=vs, simplification_factor=simplification_factor,
                              max_simplification_error=max_simplification_error, skip_ids=None if shard else skip_ids)
            writer.write(meshes, seg.voxel_offset, seg.shape[-3:], skip_ids=skip_ids)
            task["log"]["timer"][name] = time() - start
        yield task


@main.command("skeletonize")
@click.option("--name", type=str, default="skeletonize", help="name of operator")
@click.option("--input-chunk-name", "-i", type=str, default="chunk", help="name of the segmentation chunk to skeletonize.")
@click.option("--voxel-size", "-v", type=click.FLOAT, nargs=3, default=None, callback=default_none,
              help="voxel size of the segmentation, zyx order (default: the chunk's).")
@click.option("--output-path", "-o", type=str, default="file:///tmp/skeleton/",
              help="output path of the skeleton fragments: a local directory or file:// URL.")
@click.option("--output-format", "-t", type=click.Choice(["precomputed", "swc"]), default="precomputed", help="fragment format.")
@click.option("--scale", type=click.FLOAT, default=4, help="invalidation radius: scale * distance to boundary + const.")
@click.option("--const", type=click.FLOAT, default=500, help="invalidation radius: scale * distance to boundary + const (nm).")
@click.option("--pdrf-scale", type=click.FLOAT, default=100000, help="penalty field scale.")
@click.option("--pdrf-exponent", type=click.INT, default=4, help="penalty field exponent (1 to 16).")
@click.option("--dust-threshold", type=click.INT, default=1000, help="components with fewer voxels are not skeletonized.")
@click.option("--skip-ids", "-s", type=str, default=None, help="ids not to skeletonize, separated by commas.")
@click.option("--fill-holes/--no-fill-holes", default=False,
              help="fill every object's holes first (fill-segmentation-holes --mode remove-enclosed).")
@operator
def skeletonize(tasks, name, input_chunk_name, voxel_size, output_path, output_format, scale, const, pdrf_scale, pdrf_exponent,
                dust_threshold, skip_ids, fill_holes=False):
    """(extension) TEASAR skeletons of every object of a segmentation chunk on the GPU, written as ``{id}:{bbox}`` fragments
    (reference plugins/skeletonize.py -> kimimaro; rules restated in oracle/skeleton_oracle.py, not kimimaro's skeletons).  A
    host chunk is uploaded for the call, a GPU-resident one is skeletonized where it is."""
    from chunkflow_b200.flow.skeleton import write_fragments
    if skip_ids is not None:
        skip_ids = sorted(set(map(int, skip_ids.split(","))))
    for task in tasks:
        if task is not None:
            start = time()
            seg = task[input_chunk_name]
            dev, _ = _on_device(seg, "cuda:0")
            vs = voxel_size if voxel_size is not None else tuple(seg.voxel_size)
            skels = dev.skeletonize(voxel_size=vs, scale=scale, const=const, pdrf_scale=pdrf_scale, pdrf_exponent=pdrf_exponent,
                                    dust_threshold=dust_threshold, skip_ids=skip_ids, fill_holes=fill_holes)
            write_fragments(skels, output_path, tuple(seg.voxel_offset), seg.shape[-3:], vs, output_format)
            task["log"]["timer"][name] = time() - start
        yield task


@main.command("aggregate-skeleton-fragments")
@click.option("--name", type=str, default="aggregate-skeleton-fragments", help="name of operator")
@click.option("--input-name", "-i", type=str, default="prefix", help="input prefix name in task stream.")
@click.option("--prefix", "-p", type=str, default=None, help="prefix of skeleton fragments.")
@click.option("--fragments-path", "-f", type=str, required=True, help="storage path of skeleton fragments.")
@click.option("--output-path", "-o", type=str, default=None, help="storage path of aggregated skeletons.")
@operator
def aggregate_skeleton_fragments(tasks, name, input_name, prefix, fragments_path, output_path):
    """Merge skeleton fragments (reference flow/flow.py:623-650): the fragments of every id are concatenated, equal vertices
    merged and duplicate edges dropped.  kimimaro.postprocess (dust and tick removal, joining) is not applied."""
    from chunkflow_b200.flow.skeleton import aggregate_fragments
    if output_path is None:
        output_path = fragments_path
    if prefix:
        aggregate_fragments(fragments_path, output_path, prefix)
    for task in tasks:
        if task is not None and not prefix:
            start = time()
            aggregate_fragments(fragments_path, output_path, task[input_name])
            task["log"]["timer"][name] = time() - start
        yield task


if __name__ == "__main__":
    main()
