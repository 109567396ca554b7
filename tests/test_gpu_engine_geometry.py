"""Every entry point that takes a chunk shape refuses the same bad shapes with ERR_INVALID_ARGUMENT: a chunk smaller than
the input patch, an output crop margin that leaves no output, and a dimension beyond int32 (the last one only where no
device memory is involved).  None of these calls reaches a kernel with work: the device buffers below still hold C channels
of the whole chunk, more than any of them could ask for."""
import numpy as np
import pytest

from chunkflow_b200 import _native

pytestmark = pytest.mark.gpu

PATCH, OVERLAP, C = (8, 32, 32), (2, 8, 8), 2
MARGIN = (5, 17, 17)  # a (12, 40, 40) chunk keeps a (2, 6, 6) output
SMALL = [(7, 40, 40), (12, 31, 40), (12, 40, 31), (0, 0, 0)]  # (0, 0, 0): the shape an empty cache holds
SWALLOWED = [(10, 40, 40), (12, 34, 40), (12, 40, 34),  # no output voxel left on one axis
             (8, 40, 40), (12, 32, 40), (12, 40, 32)]   # a negative output size on one axis
HUGE = [(2 ** 32 + 40, 40, 40), (12, 2 ** 32 + 40, 40), (12, 40, 2 ** 32 + 40)]


def _engine(margin):
    return _native.Engine(input_patch_size=PATCH, output_patch_size=PATCH, output_patch_overlap=OVERLAP,
                          output_crop_margin=margin, num_output_channels=C, framework=_native.FRAMEWORK_IDENTITY)


def _entry_points(eng, shape, device=True):
    calls = {"patch_grid": lambda: eng.patch_grid(shape), "output_shape": lambda: eng.output_shape(shape)}
    if device:
        import torch
        n = max(1, int(np.prod(shape)))  # never a null pointer, which would be refused before the shape is looked at
        chunk = np.zeros(shape, np.uint8)
        d_in = torch.zeros(n, dtype=torch.uint8, device="cuda")
        d_out = torch.zeros(C * n, dtype=torch.float32, device="cuda")
        d_w = torch.zeros(n, dtype=torch.float32, device="cuda")
        calls.update(
            infer_chunk_device=lambda: eng.infer_chunk_device(d_in.data_ptr(), np.uint8, shape, d_out.data_ptr()),
            infer_slab_device=lambda: eng.infer_slab_device(d_in.data_ptr(), np.uint8, shape, 0, 1, d_out.data_ptr(),
                                                            d_w.data_ptr()),
            weight_volume_device=lambda: eng.weight_volume_device(shape, 0, 0, d_w.data_ptr()),
            plugin_begin=lambda: eng.plugin_begin(chunk))
    return calls


def _not_refused(calls):
    """The entry points that do not refuse the shape with ERR_INVALID_ARGUMENT, and what they did instead."""
    got = {}
    for name, call in calls.items():
        try:
            call()
            got[name] = "accepted"
        except _native.NativeError as err:
            if err.code != _native.ERR_INVALID_ARGUMENT:
                got[name] = err.code
    return got


@pytest.mark.parametrize("shape", SMALL)
def test_chunk_smaller_than_the_input_patch(shape):
    assert _not_refused(_entry_points(_engine((0, 0, 0)), shape)) == {}


@pytest.mark.parametrize("shape", SWALLOWED)
def test_crop_margin_that_leaves_no_output(shape):
    eng = _engine(MARGIN)
    assert eng.output_shape((12, 40, 40)) == (C, 2, 6, 6)
    assert _not_refused(_entry_points(eng, shape)) == {}


@pytest.mark.parametrize("shape", HUGE)
def test_dimension_beyond_int32(shape):
    assert _not_refused(_entry_points(_engine((0, 0, 0)), shape, device=False)) == {}
