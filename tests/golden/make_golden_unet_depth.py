"""Golden vectors of the 2- and 4-level U-Nets through the REAL reference's ``-f pytorch`` CPU path (imported with stubbed
I/O modules, see oracle/reference_harness.py).  Run in the build container:

    python tests/golden/make_golden_unet_depth.py

Writes ``unet_depth_small.npz``: per depth d, the input chunk (``input{d}``), the reference's output (``output{d}``) and the
sha256 of the seeded state dict (``state_sha256_{d}``, ``create_model(depth=d, seed=SEED)`` of unet3l.py), which the tests
rebuild instead of storing the weights.
"""
import io
import os
import sys
import tempfile
from contextlib import redirect_stdout

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from oracle.reference_harness import import_reference  # noqa: E402
from make_golden import MODEL_FILE, state_dict_digest  # noqa: E402

SEED = 5
PATCH, OVERLAP, CHANNELS = (8, 32, 32), (2, 8, 8), 3
CHUNK = (12, 40, 48)


def main():
    import torch
    torch.cuda.is_available = lambda: False  # the reference moves to CUDA whenever it can (pytorch.py:41-46)
    Inferencer, Chunk, _ = import_reference()
    from chunkflow_b200.lib import load_source
    model_src = load_source(MODEL_FILE)
    rng = np.random.default_rng(20261017)
    arrays = {}
    with tempfile.TemporaryDirectory() as tmp:
        for depth in (2, 4):
            state = model_src.create_model(cout=CHANNELS, seed=SEED, depth=depth).state_dict()
            ckpt = os.path.join(tmp, f"unet{depth}.pt")
            torch.save(state, ckpt)
            img = rng.integers(0, 256, size=CHUNK, dtype=np.uint8)
            with redirect_stdout(io.StringIO()):
                with Inferencer(MODEL_FILE, ckpt, PATCH, output_patch_overlap=OVERLAP, num_output_channels=CHANNELS,
                                batch_size=1, framework="pytorch", mask_output_chunk=True) as inf:
                    out = inf(Chunk(img))
                    assert inf.patch_inferencer.model.depth == depth
                    digest = state_dict_digest(inf.patch_inferencer.model.state_dict())
            assert digest == state_dict_digest(state)
            arrays[f"input{depth}"] = img
            arrays[f"output{depth}"] = out.array
            arrays[f"state_sha256_{depth}"] = np.array(digest)
    arrays["torch"] = np.array(torch.__version__)
    np.savez_compressed(os.path.join(HERE, "unet_depth_small.npz"), **arrays)
    print("golden vectors written to", os.path.join(HERE, "unet_depth_small.npz"))


if __name__ == "__main__":
    main()
