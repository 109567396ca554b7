"""A chunk that lives in GPU memory between operators (SURVEY.md section 8 f3).

``DeviceChunk`` wraps a CUDA ``torch.Tensor`` (the memory container only) with the ``voxel_offset`` / ``voxel_size``
bookkeeping of the reference's ``Chunk`` and mirrors, name for name, the reference methods that sit either side of the
``inference`` operator in a pipeline -- each one a hand-written kernel behind the C ABI (``include/chunkflow_b200.h``,
``csrc/operators.cu``), bit-identical to the reference's numpy code:

    normalize_contrast   reference chunk/image/base.py:93-132          (Image)
    maskout              reference chunk/base.py:811-829                (Chunk; ``mask.maskout(chunk)`` modifies ``chunk``)
    crop_margin          reference chunk/base.py:691-726                (Chunk)
    quantize             reference chunk/affinity_map/base.py:33-57     (AffinityMap)
    connected_component  reference chunk/base.py:128-137                (Chunk -> cc3d)
    agglomerate          reference plugins/agglomerate.py:8-48          (plugin -> waterz)
    evaluate             reference chunk/segmentation.py:33-67          (Segmentation -> gala, lib/gala/evaluate.py)
    remap, mask_fragments, mask_except
                         reference chunk/segmentation.py:69-109         (Segmentation -> fastremap)
    gaussian_filter_2d   reference chunk/base.py:846-853                (Chunk -> scipy.ndimage.gaussian_filter)
    median_filter        reference plugins/median_filter.py:4-7         (plugin -> scipy.ndimage.median_filter)
    clahe                reference plugins/clahe.py                     (plugin -> cv2.createCLAHE(...).apply)
    mesh                 reference flow/mesh.py                         (MeshOperator -> zmesh; rules restated)
    skeletonize          reference plugins/skeletonize.py               (plugin -> kimimaro; rules restated)
    fill_holes           reference plugins/fill_segmentation_holes.py   (plugin -> fill_voids; rules restated)

so that ``create-chunk | normalize-contrast | inference | crop-margin | quantize`` moves the image to the GPU once and
brings a uint8 thumbnail (or nothing) back instead of the 12-byte-per-voxel affinity map.  There is no CPU fallback.
"""
from __future__ import annotations

import re
from typing import NamedTuple, Optional, Sequence

import numpy as np

from .. import _native
from ..lib.cartesian_coordinate import Cartesian, to_cartesian
from .base import Chunk


def _torch():
    import torch
    if not torch.cuda.is_available():
        raise RuntimeError("chunkflow_b200.DeviceChunk needs a CUDA device (there is no CPU fallback)")
    return torch


def _dtype_code(t) -> int:
    torch = _torch()
    if t.dtype in (torch.uint8, torch.bool):
        return _native.DTYPE_U8
    if t.dtype == torch.float32:
        return _native.DTYPE_F32
    raise TypeError(f"DeviceChunk operators support uint8/bool and float32, got {t.dtype}")


def mask_array_for(chunk_dtype, mask: np.ndarray) -> np.ndarray:
    """Host-side conversion of a mask of any dtype numpy accepts in ``chunk *= mask`` (reference chunk/base.py:811-829)
    to one of the two mask dtypes the kernel takes, WITHOUT changing the result:

    * uint8 chunk: numpy multiplies in the wider unsigned type and casts back modulo 256, which equals multiplying by
      ``mask mod 256`` -> uint8 mask (signed / float masks are refused by numpy's 'same_kind' rule, and here);
    * float32 chunk: an integer mask is converted by numpy to float64, the product rounded to float32; for |mask| < 2**24
      that is the float32 product with the exactly converted mask -> float32 mask.  float64 masks are refused (the
      double-precision product does not round like a float32 one)."""
    chunk_dtype = np.dtype(chunk_dtype)
    mask = np.asarray(mask)
    if mask.dtype in (np.dtype(np.uint8), np.dtype(bool)) or (mask.dtype == np.float32 and chunk_dtype == np.float32):
        return np.ascontiguousarray(mask)
    if chunk_dtype == np.uint8:
        if mask.dtype.kind != "u":
            raise TypeError(f"numpy cannot cast {mask.dtype} to uint8 in place (same_kind); neither do we")
        return np.ascontiguousarray(mask.astype(np.uint8))  # wraps modulo 256
    if chunk_dtype == np.float32:
        if mask.dtype.kind not in "ui":
            raise TypeError(f"a {mask.dtype} mask on a float32 chunk is not supported (product rounds differently)")
        if mask.size and int(np.abs(mask.astype(np.int64)).max()) >= 2 ** 24:
            raise TypeError("integer mask values must be below 2**24 to be exact in float32")
        return np.ascontiguousarray(mask.astype(np.float32))
    raise TypeError(f"unsupported chunk dtype {chunk_dtype}")


def selected_ids(selected_obj_ids) -> Optional[np.ndarray]:
    """The id selection of Segmentation.mask_except (reference chunk/segmentation.py:92-107) as a uint64 array, or None when
    nothing is selected: a list / set / array of ids, a string like "34,45,56", or a path ending in ``.json`` that is read as
    a LOCAL file holding a list (the reference goes through CloudFiles; paths with a protocol are refused).  Negative ids
    stand for their uint64 bit pattern, the repository's convention for signed label volumes."""
    if selected_obj_ids is None:
        return None
    if isinstance(selected_obj_ids, np.ndarray) and selected_obj_ids.dtype.kind in "ui":
        return np.ascontiguousarray(selected_obj_ids.ravel().astype(np.uint64))
    if isinstance(selected_obj_ids, str) and selected_obj_ids.endswith('.json'):
        if '://' in selected_obj_ids and not selected_obj_ids.startswith('file://'):
            raise ValueError(f"only a local json file can hold the selected ids, not {selected_obj_ids}")
        import json
        with open(selected_obj_ids[len('file://'):] if selected_obj_ids.startswith('file://') else selected_obj_ids) as f:
            selected_obj_ids = set(json.load(f))
        assert len(selected_obj_ids) > 0                                  # reference segmentation.py:102
        print(f'number of selected objects: {len(selected_obj_ids)}')   # :103
    elif isinstance(selected_obj_ids, str):
        selected_obj_ids = set(int(i) for i in selected_obj_ids.split(','))   # :107
    ids = [int(i) for i in np.asarray(list(selected_obj_ids), dtype=object).ravel()]
    if any(not -2 ** 63 <= i < 2 ** 64 for i in ids):
        raise ValueError("a selected id does not fit in 64 bits")
    return np.array([i % 2 ** 64 for i in ids], dtype=np.uint64)


def gaussian_weights(sigma) -> np.ndarray:
    """float64 weights w[0..radius] (w[0] the centre) of scipy.ndimage's gaussian kernel at truncate 4.  Computed here with
    numpy, with scipy's own expression, and handed to the kernel: numpy's exp and the C library's may differ in the last bit,
    and one bit in a weight can change a truncated uint8 result."""
    sigma = float(sigma)
    radius = int(4.0 * sigma + 0.5)
    x = np.arange(-radius, radius + 1)
    w = np.exp(-0.5 / sigma ** 2 * x ** 2)
    w = w / w.sum()
    return np.ascontiguousarray(w[radius:])


def _per_axis(value, ndim, kind=float) -> list:
    """A scalar or one value per axis, like scipy.ndimage's _normalize_sequence (RuntimeError on another length)."""
    v = np.asarray(value)
    if v.ndim == 0:
        return [kind(v)] * ndim
    if v.ndim != 1 or v.size != ndim:
        raise RuntimeError("sequence argument must have length equal to input rank")
    return [kind(e) for e in v]


def _filter_code(t) -> int:
    torch = _torch()
    if t.dtype == torch.uint8:
        return _native.DTYPE_U8
    if t.dtype == torch.float32:
        return _native.DTYPE_F32
    raise TypeError(f"the filters take uint8 or float32 chunks, not {t.dtype}")


def _grown_table(device, slots: int, workspace_bytes, build, what: str):
    """(workspace, slots, entries) of a caller-sized hash table: ``build(workspace, slots)`` returns the number of entries or
    raises ERR_CAPACITY; the table is rebuilt four times as large while it is too full or more than half full (long probe
    sequences)."""
    torch = _torch()
    while True:
        work = torch.empty(workspace_bytes(slots), dtype=torch.uint8, device=device)
        try:
            n = build(work, slots)
            if 2 * n <= slots:
                return work, slots, n
        except _native.NativeError as err:
            if err.code != _native.ERR_CAPACITY:
                raise
        del work
        slots <<= 2
        if slots >= 1 << 31:
            raise RuntimeError(f"{what} than the table can hold")


MEAN_AFFINITY = 'OneMinus<MeanAffinity<RegionGraphType, ScoreValue>>'
_HIST_QUANTILE = re.compile(r'OneMinus<HistogramQuantileAffinity<RegionGraphType,([+-]?\d+),ScoreValue,([+-]?\d+)(?:,(\w+))?>>')


class HistogramQuantile(NamedTuple):
    """``OneMinus<HistogramQuantileAffinity<RegionGraphType, quantile, ScoreValue, bins, init_with_max>>``"""
    quantile: int
    bins: int
    init_with_max: bool


def parse_scoring_function(scoring_function: str) -> Optional[HistogramQuantile]:
    """None for waterz's mean affinity, a :class:`HistogramQuantile` for its histogram-quantile family (whitespace ignored;
    an omitted init_with_max means true, waterz's default).  Any other scoring function raises NotImplementedError, one of the
    family with a quantile outside 0..100, bins outside 2..256 or init_with_max other than true / false ValueError."""
    s = re.sub(r'\s', '', scoring_function) if isinstance(scoring_function, str) else None
    if s == MEAN_AFFINITY.replace(' ', ''):
        return None
    m = _HIST_QUANTILE.fullmatch(s) if s is not None else None
    if m is None:
        raise NotImplementedError(f'scoring function {scoring_function!r}: only {MEAN_AFFINITY} and '
                                  'OneMinus<HistogramQuantileAffinity<RegionGraphType, Q, ScoreValue, B[, I]>> are implemented')
    q, bins, init = int(m.group(1)), int(m.group(2)), m.group(3)
    if not 0 <= q <= 100:
        raise ValueError(f'the quantile must be in 0..100, not {q}')
    if not 2 <= bins <= 256:
        raise ValueError(f'the number of bins must be in 2..256, not {bins}')
    if init not in (None, 'true', 'false'):
        raise ValueError(f'init_with_max must be true or false, not {init}')
    return HistogramQuantile(q, bins, init != 'false')


class DeviceChunk:
    def __init__(self, tensor, voxel_offset=None, voxel_size=None, layer_type: Optional[str] = None):
        torch = _torch()
        assert isinstance(tensor, torch.Tensor) and tensor.is_cuda, "DeviceChunk wraps a CUDA tensor"
        assert tensor.ndim in (3, 4)
        self.tensor = tensor.contiguous()
        self.voxel_offset = to_cartesian(voxel_offset) if voxel_offset is not None else Cartesian(0, 0, 0)
        self.voxel_size = to_cartesian(voxel_size) if voxel_size is not None else None
        self.layer_type = layer_type

    # ---- host <-> device -------------------------------------------------------------------
    @classmethod
    def from_chunk(cls, chunk: Chunk, device="cuda:0") -> "DeviceChunk":
        torch = _torch()
        arr = np.ascontiguousarray(chunk.array)
        return cls(torch.from_numpy(arr).to(device), voxel_offset=chunk.voxel_offset, voxel_size=chunk.voxel_size,
                   layer_type=getattr(chunk, "_layer_type", None))

    @classmethod
    def mask_from_chunk(cls, mask: Chunk, like: "DeviceChunk") -> "DeviceChunk":
        """A mask chunk of any numpy dtype (the reference's own test uses uint32) for ``maskout`` of ``like``:
        converted on the host by :func:`mask_array_for`, then uploaded to ``like``'s GPU."""
        torch = _torch()
        target = np.uint8 if like.tensor.dtype == torch.uint8 else np.float32
        arr = mask_array_for(target, mask.array)
        return cls(torch.from_numpy(arr).to(like.tensor.device), voxel_offset=mask.voxel_offset, voxel_size=mask.voxel_size)

    def to_chunk(self) -> Chunk:
        return Chunk(self.tensor.cpu().numpy(), voxel_offset=self.voxel_offset, voxel_size=self.voxel_size)

    @property
    def shape(self):
        return tuple(self.tensor.shape)

    @property
    def dtype(self):
        return self.tensor.dtype

    @property
    def is_image(self) -> bool:
        """uint8 and 3-D, like the reference's Chunk.is_image."""
        return self.tensor.dtype == _torch().uint8 and self.tensor.ndim == 3

    def _czyx(self):
        s = self.shape
        return (1,) + s if len(s) == 3 else s

    def _stream(self) -> int:
        return _torch().cuda.current_stream(self.tensor.device).cuda_stream

    def _on_device(self):
        return _torch().cuda.device(self.tensor.device)

    # ---- Image.normalize_contrast ---------------------------------------------------------
    def normalize_contrast(self, lower_clip_fraction: float = 0.01, upper_clip_fraction: float = 0.01, minval: int = 1,
                           maxval: int = 255, per_section: bool = True) -> None:
        """In place, like the reference (including its quirks: the whole-array pass also runs after the per-section pass,
        and ``per_section=False`` does nothing)."""
        torch = _torch()
        assert self.tensor.dtype == torch.uint8 and self.tensor.ndim == 3, "normalize_contrast works on a (z,y,x) uint8 image"
        with self._on_device():
            _native.normalize_contrast_device(self.tensor.data_ptr(), self.shape, lower_clip_fraction, upper_clip_fraction,
                                              minval, maxval, per_section, self._stream())

    # ---- Chunk.maskout: self is the MASK, ``chunk`` is modified in place ---------------------
    def maskout(self, chunk: "DeviceChunk") -> None:
        assert chunk.voxel_size is not None and self.voxel_size is not None  # reference chunk/base.py:814-815
        assert all(m >= c for m, c in zip(self.voxel_size, chunk.voxel_size))
        assert all(m % c == 0 for m, c in zip(self.voxel_size, chunk.voxel_size)), "the voxel size should be divisible"
        factor = tuple(m // c for m, c in zip(self.voxel_size, chunk.voxel_size))
        assert self.tensor.ndim == 3
        assert tuple(chunk.shape[-3:]) == tuple(s * f for s, f in zip(self.shape, factor)), \
            "chunk size must equal mask size times the voxel-size factor"
        with self._on_device():
            _native.maskout_device(chunk.tensor.data_ptr(), _dtype_code(chunk.tensor), chunk._czyx(), self.tensor.data_ptr(),
                                   _dtype_code(self.tensor), factor, chunk._stream())

    # ---- Chunk.crop_margin ----------------------------------------------------------------
    def crop_margin(self, margin_size: Sequence[int]) -> "DeviceChunk":
        torch = _torch()
        m = tuple(int(v) for v in margin_size)
        if len(m) == 3:
            m6 = m + m
        elif len(m) == 6:
            m6 = m
        else:
            raise ValueError('only support 3 or 6 elements.')  # reference chunk/base.py:719
        c, z, y, x = self._czyx()
        out_sp = (z - m6[0] - m6[3], y - m6[1] - m6[4], x - m6[2] - m6[5])
        out_shape = out_sp if self.tensor.ndim == 3 else (c,) + out_sp
        dst = torch.empty(out_shape, dtype=self.tensor.dtype, device=self.tensor.device)
        with self._on_device():
            _native.crop_margin_device(self.tensor.data_ptr(), _dtype_code(self.tensor), (c, z, y, x), m6, dst.data_ptr(),
                                       self._stream())
        offset = tuple(o + mm for o, mm in zip(self.voxel_offset, m))  # the three lower margins (reference :721-722)
        return DeviceChunk(dst, voxel_offset=offset, voxel_size=self.voxel_size)

    # ---- AffinityMap.quantize -------------------------------------------------------------
    def quantize(self, mode: str = 'xy') -> "DeviceChunk":
        torch = _torch()
        assert self.tensor.dtype == torch.float32 and self.tensor.ndim == 4, "quantize works on a (c,z,y,x) float32 affinity map"
        if mode == 'xy':
            code = _native.QUANTIZE_XY
        elif mode == 'z':
            code = _native.QUANTIZE_Z
        else:
            raise ValueError(f'only support xy and z mode, but got {mode}')
        out = torch.empty(self.shape[1:], dtype=torch.uint8, device=self.tensor.device)
        with self._on_device():
            _native.quantize_device(self.tensor.data_ptr(), self.shape, code, out.data_ptr(), self._stream())
        return DeviceChunk(out, voxel_offset=self.voxel_offset, voxel_size=self.voxel_size)

    # ---- Chunk.connected_component ---------------------------------------------------------
    def connected_component(self, threshold: float = None, connectivity: int = 6) -> "DeviceChunk":
        """Threshold the map and label its connected components (reference chunk/base.py:128-137: ``Chunk.threshold`` --
        ``array > threshold`` -- for non-segmentation chunks, then ``cc3d.connected_components(seg, connectivity)``).
        (z,y,x) or (1,z,y,x) float32 map with a threshold, or a uint8 / int32 / uint32 segmentation; returns a (z,y,x) uint32
        segmentation whose components are numbered 1..N in raster order of their first voxel, like cc3d."""
        torch = _torch()
        t = self.tensor
        if t.ndim == 4:
            assert t.shape[0] == 1   # reference base.py:730-732
            t = t[0]
        is_seg = t.dtype in (torch.uint8, torch.bool, torch.int32, torch.uint32) or self.layer_type == "segmentation"
        thr = 0.0
        if not is_seg and threshold is not None:
            assert t.dtype == torch.float32, "thresholding works on a float32 map"
            code, thr = _native.DTYPE_F32, float(threshold)
        elif t.dtype in (torch.uint8, torch.bool):
            code = _native.DTYPE_U8
        elif t.dtype in (torch.int32, torch.uint32):
            code = _native.DTYPE_U32
        else:
            raise TypeError(f"connected_component: {t.dtype} without a threshold is not a segmentation (uint8 / int32 / uint32)")
        if connectivity not in (6, 18, 26):
            raise ValueError("connectivity must be 6, 18 or 26")
        t = t.contiguous()
        labels = torch.empty(t.shape, dtype=torch.int32, device=t.device)   # uint32 values (torch has no full uint32 support)
        work = torch.empty(_native.connected_components_workspace(t.shape), dtype=torch.uint8, device=t.device)
        with self._on_device():
            self.num_components = _native.connected_components_device(t.data_ptr(), code, tuple(t.shape), thr, connectivity,
                                                                      labels.data_ptr(), work.data_ptr(), self._stream())
        del work
        out = DeviceChunk(labels.view(torch.uint32) if hasattr(torch, "uint32") else labels, voxel_offset=self.voxel_offset,
                          voxel_size=self.voxel_size, layer_type="segmentation")
        out.num_components = self.num_components
        return out

    # ---- plugins/agglomerate.py: watershed fragments + mean-affinity agglomeration --------------
    def _affinity_tensor(self):
        torch = _torch()
        t = self.tensor
        assert t.ndim == 4 and t.shape[0] == 3 and t.dtype == torch.float32, \
            "an affinity map is a (3, z, y, x) float32 chunk (the reference converts with np.ascontiguousarray(affs, dtype=float32))"
        if t.numel() // 3 >= 2 ** 32 - 1:
            raise ValueError("more than 2^32 - 1 voxels")
        return t

    def watershed(self, aff_threshold_low: float = 0.001, aff_threshold_high: float = 0.9999,
                  flip_channel: bool = True) -> "DeviceChunk":
        """Fragments of the affinity map by steepest-ascent watershed (what ``waterz.agglomerate`` computes first when no
        fragments are passed, reference plugins/agglomerate.py:36-41): (z,y,x) uint32, basins numbered 1..N in raster order
        of their first voxel, 0 where no affinity exceeds ``aff_threshold_low``.  ``flip_channel``: the channels are stored
        in chunkflow's order x, y, z (agglomerate.py:26-29); they are read in reverse, not copied."""
        torch = _torch()
        t = self._affinity_tensor()
        zyx = tuple(t.shape[1:])
        frag = torch.empty(zyx, dtype=torch.int32, device=t.device)   # uint32 values
        work = torch.empty(_native.watershed_workspace(zyx), dtype=torch.uint8, device=t.device)
        with self._on_device():
            n = _native.watershed_device(t.data_ptr(), flip_channel, zyx, aff_threshold_low, aff_threshold_high, frag.data_ptr(),
                                         work.data_ptr(), self._stream())
        del work
        out = DeviceChunk(frag.view(torch.uint32) if hasattr(torch, "uint32") else frag, voxel_offset=self.voxel_offset,
                          voxel_size=self.voxel_size, layer_type="segmentation")
        out.num_components = n
        return out

    def region_graph(self, fragments: "DeviceChunk", flip_channel: bool = True, num_fragments: Optional[int] = None,
                     histogram_bins: Optional[int] = None):
        """(u, v, sum_fixed, count) host arrays, one entry per pair of touching fragments, sorted by (u, v): the sum (2^-30
        fixed point) and number of the affinities on the faces between them (waterz's region graph with MeanAffinity
        statistics).  The hash table is sized from the fragment count and grown on overflow.

        With ``histogram_bins`` B (2..256): (u, v, offsets, bins, counts, maxima) instead, the statistics of waterz's
        HistogramQuantileAffinity -- edge i counts ``counts[offsets[i]:offsets[i+1]]`` faces in the increasing ``bins`` of
        the same slice (bin = min(int(a * B), B - 1) of the clamped affinity, float32), and ``maxima[i]`` is its largest
        clamped affinity."""
        torch = _torch()
        t = self._affinity_tensor()
        f = fragments.tensor
        assert tuple(f.shape) == tuple(t.shape[1:]) and f.dtype in (torch.int32, torch.uint32) and f.device == t.device
        if num_fragments is None:
            num_fragments = getattr(fragments, "num_components", None)
        if num_fragments is None:
            num_fragments = int(f.view(torch.int32).max().item()) if f.numel() else 0
        slots = 1 << 16
        while slots < 16 * num_fragments:
            slots <<= 1
        if histogram_bins is not None:
            return self._region_graph_hist(t, f, flip_channel, int(histogram_bins), slots)
        with self._on_device():
            work, slots, n = _grown_table(
                t.device, slots, _native.region_graph_workspace,
                lambda work, slots: _native.region_graph_device(t.data_ptr(), flip_channel, f.data_ptr(), tuple(f.shape),
                                                                work.data_ptr(), slots, self._stream()),
                "region graph: more fragment pairs")
            return _native.region_graph_read(work.data_ptr(), slots, n, self._stream())

    def _region_graph_hist(self, t, f, flip_channel, bins, slots):
        found = {}

        def build(work, slots):
            found["edges"], found["entries"] = _native.region_graph_hist_device(
                t.data_ptr(), flip_channel, f.data_ptr(), tuple(f.shape), bins, work.data_ptr(), slots, self._stream())
            # the bin table has HIST_SLOTS_PER_SLOT times as many slots: keep both at most half full
            return max(found["edges"], -(-found["entries"] // _native.HIST_SLOTS_PER_SLOT))

        with self._on_device():
            work, slots, _ = _grown_table(t.device, slots, _native.region_graph_hist_workspace, build,
                                          "region graph: more fragment pairs or histogram bins")
            return _native.region_graph_hist_read(work.data_ptr(), slots, found["edges"], found["entries"], self._stream())

    def agglomerate(self, threshold: float = 0.7, aff_threshold_low: float = 0.001, aff_threshold_high: float = 0.9999,
                    fragments: Optional["DeviceChunk"] = None, flip_channel: bool = True,
                    scoring_function: str = MEAN_AFFINITY) -> "DeviceChunk":
        """Agglomeration including the watershed step (reference plugins/agglomerate.py:8-48 -> ``waterz.agglomerate``):
        fragments (watershed, unless given) -> region graph -> merge edges in order of increasing score until
        ``threshold`` -> relabel.  ``scoring_function``: waterz's ``OneMinus<MeanAffinity<RegionGraphType, ScoreValue>>``
        (1 - mean affinity) or ``OneMinus<HistogramQuantileAffinity<RegionGraphType, Q, ScoreValue, B[, I]>>`` (1 - the
        Q-th percentile of a B-bin histogram of the affinities; with I, 1 - the largest affinity until an edge is pooled),
        see :func:`parse_scoring_function`.  The voxel passes are CUDA kernels; the merge loop over the fragment graph runs
        in the native library on the host (as waterz's does).  Returns a (z,y,x) uint32 segmentation whose ids are the
        surviving fragment ids."""
        torch = _torch()
        hq = parse_scoring_function(scoring_function)
        t = self._affinity_tensor()
        if fragments is None:
            fragments = self.watershed(aff_threshold_low, aff_threshold_high, flip_channel)
        f = fragments.tensor
        if f.dtype not in (torch.int32, torch.uint32):
            raise TypeError("fragments must be an int32 / uint32 segmentation on the device")
        num = getattr(fragments, "num_components", None)
        if num is None:
            num = int(f.view(torch.int32).max().item()) if f.numel() else 0
        if num < 0:
            raise ValueError("fragment ids must be below 2^31")
        if hq is None:
            u, v, s, c = self.region_graph(fragments, flip_channel, num)
            root = _native.agglomerate_edges_host(num + 1, u, v, s, c, threshold)
        else:
            u, v, off, b, c, mx = self.region_graph(fragments, flip_channel, num, histogram_bins=hq.bins)
            root = _native.agglomerate_quantile_host(num + 1, u, v, off, b, c, mx, threshold, hq.quantile, hq.bins, hq.init_with_max)
        d_root = torch.from_numpy(root.view(np.int32)).to(t.device)
        seg = torch.empty(f.shape, dtype=torch.int32, device=t.device)
        with self._on_device():
            _native.relabel_device(f.data_ptr(), f.numel(), d_root.data_ptr(), root.size, seg.data_ptr(), self._stream())
            _torch().cuda.current_stream(t.device).synchronize()   # d_root is released below
        out = DeviceChunk(seg.view(torch.uint32) if hasattr(torch, "uint32") else seg, voxel_offset=self.voxel_offset,
                          voxel_size=self.voxel_size, layer_type="segmentation")
        out.num_fragments, out.num_edges = num, int(u.size)
        out.num_components = int(np.count_nonzero(root[1:] == np.arange(1, root.size, dtype=np.uint32)))
        return out

    # ---- Segmentation.evaluate: contingency table + gala's scores -----------------------------------
    def _label_tensor(self):
        """(tensor, dtype code) of a (z,y,x) label volume.  Repository convention: int32 holds uint32 values and int64 the
        uint64 bit pattern (what numpy's astype(np.uint64) gives a signed array) -- every score is invariant under this
        one-to-one relabelling."""
        torch = _torch()
        t = self.tensor
        if t.ndim == 4:
            assert t.shape[0] == 1, "a segmentation has one channel"
            t = t[0]
        codes = {torch.uint8: _native.DTYPE_U8, torch.bool: _native.DTYPE_U8, torch.int32: _native.DTYPE_U32,
                 torch.int64: _native.DTYPE_U64}
        for name, code in (("uint32", _native.DTYPE_U32), ("uint64", _native.DTYPE_U64)):
            if hasattr(torch, name):
                codes[getattr(torch, name)] = code
        if t.dtype not in codes:
            raise TypeError(f"a label volume on the device is uint8, int32 / uint32 or int64 / uint64, not {t.dtype}")
        if t.numel() >= 2 ** 32 - 1:
            raise ValueError("more than 2^32 - 1 voxels")
        return t.contiguous(), codes[t.dtype]

    def _contingency(self, groundtruth: "DeviceChunk", table_slots: Optional[int] = None):
        """(workspace, slots, pairs): the contingency table of self (rows) and ``groundtruth`` (columns) built on the device.
        The table starts at ``table_slots`` (default: from the voxel count) and is grown on overflow."""
        torch = _torch()
        s, sc = self._label_tensor()
        g, gc = groundtruth._label_tensor()
        if tuple(s.shape) != tuple(g.shape) or s.device != g.device:
            raise ValueError(f"segmentation {tuple(s.shape)} and ground truth {tuple(g.shape)} must have the same shape and device")
        slots = int(table_slots) if table_slots is not None else 1 << max(10, min(24, (s.numel() // 64).bit_length()))
        with self._on_device():
            return _grown_table(
                s.device, slots, _native.evaluate_workspace,
                lambda work, slots: _native.contingency_device(s.data_ptr(), sc, g.data_ptr(), gc, tuple(s.shape), work.data_ptr(),
                                                               slots, self._stream()),
                "evaluate: more label pairs")

    def contingency_table(self, groundtruth: "DeviceChunk", table_slots: Optional[int] = None):
        """gala's contingency_table(seg, gt, norm=False) (reference lib/gala/evaluate.py:212-249) with nothing ignored:
        (seg ids uint64, gt ids uint64, voxel counts uint32) host arrays, one entry per pair that occurs, sorted by (seg, gt)."""
        work, slots, n = self._contingency(groundtruth, table_slots)
        with self._on_device():
            return _native.contingency_read(work.data_ptr(), slots, n, self._stream())

    def evaluate_statistics(self, groundtruth: "DeviceChunk", size_thresholds=(1000,), table_slots: Optional[int] = None) -> list:
        """One table, scored for every threshold of ``size_thresholds``: a list of dicts with the statistics (cfb_seg_scores)
        and the five scores.  A threshold sweep costs one voxel pass."""
        work, slots, _ = self._contingency(groundtruth, table_slots)
        with self._on_device():
            return [_native.contingency_scores(work.data_ptr(), slots, t, self._stream()).as_dict() for t in size_thresholds]

    def evaluate(self, groundtruth: "DeviceChunk", size_threshold: float = 1000, table_slots: Optional[int] = None) -> dict:
        """Segmentation.evaluate (reference chunk/segmentation.py:33-67) without its printed lines: rand index, adjusted rand
        index, variation of information, Fowlkes-Mallows index and edit distance (false merges, false splits) of self against
        ``groundtruth``, as numpy float64 like the reference's.  See include/chunkflow_b200.h for the definitions and the
        reference quirks that are kept."""
        st = self.evaluate_statistics(groundtruth, (size_threshold,), table_slots)[0]
        f = np.float64
        return {"rand_index": f(st["rand_index"]), "adjusted_rand_index": f(st["adjusted_rand_index"]),
                "variation_of_information": f(st["variation_of_information"]),
                "fowlkes_mallows_index": f(st["fowlkes_mallows_index"]),
                "edit_distance": (f(st["false_merges"]), f(st["false_splits"]))}

    # ---- Segmentation.remap / mask_fragments / mask_except: label table + one relabelling pass --------------
    def _label_table(self, table_slots: Optional[int] = None):
        """(label tensor, dtype code, workspace, slots, labels): the table id -> (voxel count, first voxel) of the volume, built
        on the device in one read.  The table starts at ``table_slots`` (default: from the voxel count) and is grown on
        overflow."""
        t, code = self._label_tensor()
        if t.numel() == 0:
            raise ValueError("an empty volume has no labels")
        n = t.numel()
        slots = int(table_slots) if table_slots is not None else 1 << max(10, min(24, (n // 64).bit_length()))
        with self._on_device():
            work, slots, num = _grown_table(
                t.device, slots, lambda slots: _native.label_table_workspace(n, slots),
                lambda work, slots: _native.label_table_device(t.data_ptr(), code, tuple(t.shape), work.data_ptr(), slots,
                                                               self._stream()),
                "label table: more labels")
        return t, code, work, slots, num

    def _label_numpy_dtype(self, code):
        return {_native.DTYPE_U8: np.uint8, _native.DTYPE_U32: np.uint32, _native.DTYPE_U64: np.uint64}[code]

    def unique(self, return_counts: bool = False, table_slots: Optional[int] = None):
        """fastremap.unique of the label volume (as the reference uses it, chunk/segmentation.py:87): the ids in ascending
        order (as unsigned values, in the volume's unsigned dtype) and, with ``return_counts``, their voxel counts (int64).
        One read of the volume; only the table comes to the host."""
        _, code, work, slots, num = self._label_table(table_slots)
        with self._on_device():
            ids, counts, _ = _native.label_table_read(work.data_ptr(), slots, num, self._stream())
        ids = ids.astype(self._label_numpy_dtype(code))
        return (ids, counts.astype(np.int64)) if return_counts else ids

    def _relabel(self, dust_threshold=None, keep_ids: Optional[np.ndarray] = None, renumber: bool = False, base_id: int = 0,
                 table_slots: Optional[int] = None):
        """Count pass, plan and apply pass (csrc/relabel.cu); the tensor is replaced by the result.  Masks keep the dtype and
        work in place; renumbering gives the uint64 bit pattern in an int64 tensor.
        -> (labels in the volume, entries failing the dust test, surviving non-zero ids, maximum of the result)."""
        torch = _torch()
        base_id = _native.check_base_id(base_id)
        t, code, work, slots, num = self._label_table(table_slots)
        shape = tuple(self.tensor.shape)
        with self._on_device():
            d_keep = None
            if keep_ids is not None and keep_ids.size:
                d_keep = torch.from_numpy(np.ascontiguousarray(keep_ids, np.uint64).view(np.int64)).to(t.device)
            dust, survivors, new_max = _native.label_table_plan(
                work.data_ptr(), slots, t.numel(), dust_threshold, d_keep.data_ptr() if d_keep is not None else 0,
                None if keep_ids is None else int(keep_ids.size), renumber, base_id, self._stream())
            out = torch.empty(t.shape, dtype=torch.int64, device=t.device) if renumber else t
            _native.label_apply_device(t.data_ptr(), code, t.numel(), work.data_ptr(), slots, out.data_ptr(),
                                       _native.DTYPE_U64 if renumber else code, self._stream())   # synchronises: d_keep may go
        self.tensor = out.view(shape)
        self.layer_type = "segmentation"
        return num, dust, survivors, new_max

    def mask_out_objects(self, dust_size_threshold: Optional[int] = None, selected_obj_ids=None,
                         table_slots: Optional[int] = None) -> tuple:
        """mask_fragments and then mask_except (the order of `mask-out-objects`, reference flow/flow.py:2044-2047) sharing one
        count pass and one relabelling pass; either may be None.  In place.  -> (labels in the volume, labels failing the dust
        test): the two numbers mask_fragments prints."""
        keep = selected_ids(selected_obj_ids)
        if dust_size_threshold is None and keep is None:
            return None
        num, dust, _, _ = self._relabel(dust_threshold=dust_size_threshold, keep_ids=keep, table_slots=table_slots)
        return num, dust

    def mask_fragments(self, voxel_num_threshold: int, table_slots: Optional[int] = None) -> tuple:
        """Segmentation.mask_fragments (reference chunk/segmentation.py:86-90) without its printed line: every id with
        ``count <= voxel_num_threshold`` becomes 0 (`<=`, like the reference's code).  In place, dtype unchanged.
        -> (labels in the volume, labels masked), 0 counted in both like the reference's line."""
        return self.mask_out_objects(dust_size_threshold=int(voxel_num_threshold), table_slots=table_slots)

    def mask_except(self, selected_obj_ids, table_slots: Optional[int] = None) -> None:
        """Segmentation.mask_except (reference chunk/segmentation.py:92-109): every id not selected becomes 0; ids that do not
        occur are ignored; an empty selection gives an all-zero volume; None does nothing.  In place, dtype unchanged."""
        self.mask_out_objects(selected_obj_ids=selected_obj_ids, table_slots=table_slots)

    def remap(self, base_id: int = 0, table_slots: Optional[int] = None) -> int:
        """Segmentation.remap (reference chunk/segmentation.py:69-84): the non-zero ids become 1..N in the order in which they
        are first met in a C-order raster scan (fastremap.renumber, preserve_zero=True), plus ``base_id``; 0 stays 0.  The
        tensor becomes the uint64 result (bit pattern in an int64 tensor).  Returns the maximum of the result, the base id of
        the next chunk -- 0 for an all-zero chunk whatever ``base_id``: the reference's value, kept."""
        return self._relabel(renumber=True, base_id=base_id, table_slots=table_slots)[3]

    # ---- `downsample`: uint8 averaging, countless mode pooling of segmentations ---------------------------------
    def downsample(self, factor=(2, 2, 2)) -> "DeviceChunk":
        """The reference's `downsample` command (flow/flow.py:1545-1573) on the device: a (z,y,x) uint8 image is averaged, a
        (z,y,x) int32 / uint32 / int64 / uint64 / bool segmentation is mode-pooled (countless) or strided level after level
        (csrc/downsample.cu; the arithmetic of the reference's vendored lib/igneous/downsample.py, see
        include/chunkflow_b200.h for the rules, the quirks kept and the refusals).  int32 holds uint32 ids and int64 the
        uint64 bit pattern.  Returns a new chunk with ``voxel_offset // factor``, ``voxel_size * factor`` and the same
        ``layer_type``; the input is not changed.  A refused factor raises ValueError before any kernel runs."""
        torch = _torch()
        f = tuple(int(v) for v in factor)
        if len(f) != 3:
            raise ValueError(f"the factor is (z, y, x), not {factor}")
        t = self.tensor
        codes = {torch.int32: _native.DTYPE_U32, torch.int64: _native.DTYPE_U64, torch.bool: _native.DTYPE_BOOL}
        for name, code in (("uint32", _native.DTYPE_U32), ("uint64", _native.DTYPE_U64)):
            if hasattr(torch, name):
                codes[getattr(torch, name)] = code
        if t.ndim != 3 or (t.dtype != torch.uint8 and t.dtype not in codes):
            raise TypeError(f'only support image or segmentation, but got: {t.dtype}')
        with self._on_device():
            if t.dtype == torch.uint8:
                shape = tuple(-(-s // k) for s, k in zip(t.shape, f)) if min(f) > 0 else None
                out = torch.empty(shape or (0,), dtype=torch.uint8, device=t.device)
                _native.downsample_average_device(t.data_ptr(), t.shape, f, out.data_ptr(), self._stream())
            else:
                code = codes[t.dtype]
                shape, work_bytes = _native.downsample_workspace(code, t.shape, f)
                out = torch.empty(shape, dtype=t.dtype, device=t.device)
                work = torch.empty(work_bytes, dtype=torch.uint8, device=t.device) if work_bytes else None
                _native.downsample_segmentation_device(t.data_ptr(), code, t.shape, f, work.data_ptr() if work is not None else 0,
                                                       out.data_ptr(), self._stream())
                del work   # the caching allocator keeps it for the stream until the levels have run
        fc = Cartesian(*f)
        return DeviceChunk(out, voxel_offset=self.voxel_offset // fc,
                           voxel_size=None if self.voxel_size is None else self.voxel_size * fc, layer_type=self.layer_type)

    # ---- Chunk.gaussian_filter_2d, plugins/median_filter.py ----------------------------------------------------------
    def gaussian_filter_2d(self, sigma=1, per_channel: bool = False) -> None:
        """In place, like the reference's Chunk.gaussian_filter_2d (chunk/base.py:846-853): for every z,
        ``scipy.ndimage.gaussian_filter(array[..., z, :, :], sigma)`` bit for bit (csrc/filter_kernels.cuh).  On a (c,z,y,x)
        chunk that section is the (c,y,x) block, so -- as in the reference -- the blur also runs across the channels, the
        channel axis reflected like the others; ``sigma`` is then a scalar or (c, y, x), on a (z,y,x) chunk a scalar or (y, x).
        ``per_channel=True`` filters every (y,x) plane on its own instead, as plugins/gaussian_filter.py does.  An axis with
        sigma <= 1e-15 is not filtered.  uint8 or float32; a radius int(4 sigma + 0.5) above 64 raises ValueError, another
        dtype TypeError, before any kernel runs."""
        torch = _torch()
        t = self.tensor
        code = _filter_code(t)
        axes = 2 if t.ndim == 3 or per_channel else 3
        weights = []
        for s in _per_axis(sigma, axes):
            w = gaussian_weights(s) if s > 1e-15 else None
            if w is not None and len(w) - 1 > _native.MAX_GAUSSIAN_RADIUS:
                raise ValueError(f"gaussian filter: radius {len(w) - 1} exceeds the limit of {_native.MAX_GAUSSIAN_RADIUS}")
            weights.append(w)
        if t.ndim == 4 and per_channel:
            weights = [None] + weights
        with self._on_device():
            work_bytes = _native.gaussian_filter_workspace(code, t.shape)
            work = torch.empty(work_bytes, dtype=torch.uint8, device=t.device)
            _native.gaussian_filter_device(t.data_ptr(), code, t.shape, weights, work.data_ptr(), work_bytes, self._stream())
            del work   # the caching allocator keeps it for the stream until the kernels have run

    def median_filter(self, size=(3, 1, 1), mode: str = "reflect") -> "DeviceChunk":
        """``scipy.ndimage.median_filter(array, size=size, mode=mode)`` bit for bit, as plugins/median_filter.py runs it
        (csrc/filter_kernels.cuh): element V // 2 of the sorted window of V elements, the window of extent s spanning offsets
        -(s // 2) .. s - 1 - (s // 2).  ``size`` is a scalar or one extent per axis of the chunk (RuntimeError otherwise,
        like scipy); ``mode`` reflect, nearest, mirror, wrap, constant (0) or a grid-* alias.  uint8 or float32, windows of at
        most 125 elements.  Returns a new chunk with the same offset, voxel size and layer type.  float32 NaN and the sign of
        a zero in a tie are outside the bit-identity claim."""
        torch = _torch()
        t = self.tensor
        code = _filter_code(t)
        extents = _per_axis(size, t.ndim, int)
        if mode not in _native.FILTER_MODES:
            raise RuntimeError(f"boundary mode not supported: {mode}")
        if min(extents) < 1:
            raise ValueError("every window extent must be at least 1")
        volume = int(np.prod(extents))
        if volume > _native.MAX_MEDIAN_WINDOW:
            raise ValueError(f"median filter: a window of {volume} elements exceeds the limit of {_native.MAX_MEDIAN_WINDOW} (5x5x5)")
        out = torch.empty_like(t)
        with self._on_device():
            _native.median_filter_device(t.data_ptr(), code, t.shape, extents, mode, out.data_ptr(), self._stream())
        return DeviceChunk(out, voxel_offset=self.voxel_offset, voxel_size=self.voxel_size, layer_type=self.layer_type)

    # ---- plugins/clahe.py ------------------------------------------------------------------------------------------------
    def clahe(self, clip_limit: float = 20.0, tile_grid_size=(512, 512)) -> "DeviceChunk":
        """``cv2.createCLAHE(clip_limit, tile_grid_size).apply`` of every z section bit for bit, as plugins/clahe.py runs it
        (csrc/clahe_kernels.cuh).  ``tile_grid_size`` is (x, y) -- OpenCV's order, x first.  A clip limit <= 0 means no
        clipping.  uint8 (z, y, x) only: another dtype raises TypeError, another ndim or fewer than one tile along an axis
        ValueError, before any kernel runs.  Returns a new chunk with the same offset, voxel size and layer type."""
        torch = _torch()
        t = self.tensor
        if t.dtype != torch.uint8:
            raise TypeError(f"clahe takes uint8 images, not {t.dtype}")
        zyx, tx, ty = _native.clahe_args(t.shape, tile_grid_size)
        out = torch.empty_like(t)
        with self._on_device():
            work_bytes = _native.clahe_workspace(zyx, (tx, ty))
            work = torch.empty(work_bytes, dtype=torch.uint8, device=t.device) if work_bytes else None
            _native.clahe_device(t.data_ptr(), out.data_ptr(), zyx, clip_limit, (tx, ty), work.data_ptr() if work_bytes else 0,
                                 work_bytes, self._stream())
            del work   # the caching allocator keeps it for the stream until the kernels have run
        return DeviceChunk(out, voxel_offset=self.voxel_offset, voxel_size=self.voxel_size, layer_type=self.layer_type)

    def _ids(self, op: str):
        """(contiguous (z, y, x) tensor, DTYPE_U32 / DTYPE_U64) of a segmentation of uint32 / int32 / uint64 / int64 ids."""
        torch = _torch()
        t = self.tensor.contiguous()
        if t.ndim != 3:
            raise ValueError(f"{op} takes a (z, y, x) segmentation, not a {t.ndim}-D chunk")
        codes = {torch.int32: _native.DTYPE_U32, torch.int64: _native.DTYPE_U64}
        for name, code in (("uint32", _native.DTYPE_U32), ("uint64", _native.DTYPE_U64)):
            if hasattr(torch, name):
                codes[getattr(torch, name)] = code
        if t.dtype not in codes:
            raise TypeError(f"{op} takes uint32, int32, uint64 or int64 ids, not {t.dtype}")
        return t, codes[t.dtype]

    def _physical_voxel_size(self, voxel_size) -> tuple:
        vs = self.voxel_size if voxel_size is None else voxel_size
        vs = tuple(float(v) for v in (vs if vs is not None else (1, 1, 1)))
        if len(vs) != 3:
            raise ValueError(f"the voxel size is (z, y, x), not {vs}")
        return vs

    # ---- `mesh`: marching cubes on the device, welding and simplification on the host --------------------------------------
    def mesh(self, voxel_size=None, simplification_factor: int = 100, max_simplification_error: float = 40, skip_ids=None,
             close: bool = False, threads: int = 0) -> dict:
        """Meshes of every object of a (z,y,x) segmentation (csrc/mesh.cu, rules in oracle/mesh_oracle.py; not zmesh's meshes):
        ``{id: (vertices float32 (N, 3) x, y, z in physical units, faces uint32 (M, 3))}`` in the chunk's own frame, ids
        ascending.  ``voxel_size`` is (z, y, x), the chunk's by default.  0 and the ``skip_ids`` are not meshed.  The mesh is
        open at the chunk faces unless ``close`` (everything outside the chunk is then 0 and every object watertight).
        ``simplification_factor`` > 1 simplifies each object towards ceil(faces / factor) faces while the error stays within
        ``max_simplification_error`` (nm, like zmesh's).  uint32 / int32 / uint64 / int64 ids (signed ones by their bit
        pattern); another dtype raises TypeError and another ndim ValueError before any kernel runs.  The meshes are welded on
        the device; ``threads``: host workers of the simplifier (0: the hardware's); the result does not depend on it."""
        torch = _torch()
        t, code = self._ids("mesh")
        if isinstance(simplification_factor, bool) or not isinstance(simplification_factor, (int, np.integer)):
            raise TypeError("the simplification factor is an integer")
        vs = self._physical_voxel_size(voxel_size)
        skip = selected_ids(skip_ids) if skip_ids is not None else np.zeros(0, np.uint64)
        skip = np.unique(skip)
        zyx = tuple(t.shape)
        if min(zyx) == 0:
            return {}
        with self._on_device():
            d_skip = torch.from_numpy(skip.view(np.int64)).to(t.device) if skip.size else None
            work = torch.empty(_native.mesh_workspace(zyx, close), dtype=torch.uint8, device=t.device)
            args = (t.data_ptr(), code, zyx, d_skip.data_ptr() if d_skip is not None else 0, skip.size, close)
            counts = _native.mesh_count_device(*args, work.data_ptr(), self._stream())
            nbytes = _native.mesh_buffer_bytes(counts)
            buf = torch.empty(nbytes, dtype=torch.uint8, device=t.device)
            n = _native.mesh_device(*args, vs, work.data_ptr(), counts, buf.data_ptr(), nbytes, self._stream())
            meshes = _native.mesh_read(buf.data_ptr(), counts, n, self._stream())
            del buf, work
        if simplification_factor <= 1 or not meshes:
            return meshes
        from concurrent.futures import ThreadPoolExecutor   # the native simplifier releases the GIL
        import os
        workers = threads if threads > 0 else min(32, os.cpu_count() or 1)
        keys = list(meshes)
        with ThreadPoolExecutor(max_workers=workers) as pool:
            out = pool.map(lambda k: _native.mesh_simplify_host(*meshes[k], simplification_factor, max_simplification_error), keys)
            return dict(zip(keys, out))

    # ---- `fill-segmentation-holes`: components and their faces on the device, enclosure on the host ---------------------------
    def fill_holes(self, mode: str = "binary", return_fill_count: bool = False, stats: Optional[dict] = None):
        """fill_voids.fill of a (z, y, x) chunk and its per-object extensions (csrc/fill_holes.cu, rules in
        oracle/fill_holes_oracle.py), 6-connected, outside = beyond the chunk's faces.  ``binary`` (the reference plugin): 1 for
        every voxel != 0 and every background voxel with no background path to outside, 0 elsewhere; bool, uint8, int32, uint32,
        int64, uint64 or float32.  ``keep-enclosed``: every 0 voxel enclosed by an object (a 6-connected component of one
        non-zero id) takes the id of the innermost one.  ``remove-enclosed``: every enclosed voxel takes the id of the outermost
        encloser.  The per-object modes take uint32 / int32 / uint64 / int64 ids (signed ones by their bit pattern).  Returns a
        new chunk in the input's dtype (and, with ``return_fill_count``, the number of voxels the rule assigned: the holes, the
        enclosed zeros, every enclosed voxel).  Another dtype, ndim or mode raises before any kernel runs.  ``stats``, when
        given, receives the components, pairs, table slots and the ms of each phase (host clock around synchronised calls)."""
        import time
        torch = _torch()
        code = _native.fill_mode(mode)
        t = self.tensor.contiguous()
        if t.ndim != 3:
            raise ValueError(f"fill holes takes a (z, y, x) chunk, not a {t.ndim}-D one")
        codes = {torch.bool: _native.DTYPE_U8, torch.uint8: _native.DTYPE_U8, torch.float32: _native.DTYPE_F32,
                 torch.int32: _native.DTYPE_U32, torch.int64: _native.DTYPE_U64}
        for name, c in (("uint32", _native.DTYPE_U32), ("uint64", _native.DTYPE_U64)):
            if hasattr(torch, name):
                codes[getattr(torch, name)] = c
        if t.dtype not in codes or (code != 0 and codes[t.dtype] not in (_native.DTYPE_U32, _native.DTYPE_U64)):
            allowed = "bool, uint8, int32, uint32, int64, uint64 or float32" if code == 0 else "uint32, int32, uint64 or int64 ids"
            raise TypeError(f"fill holes: {mode} mode takes {allowed}, not {t.dtype}")
        dtype, zyx = codes[t.dtype], tuple(t.shape)
        out = torch.empty_like(t)
        st = {"components": 0, "edges": 0, "table_slots": 0}
        count = 0
        if min(zyx) > 0:
            with self._on_device():
                s = self._stream()
                t0 = time.perf_counter()
                work = torch.empty(_native.fill_holes_workspace(zyx), dtype=torch.uint8, device=t.device)
                st["components"] = comps = _native.fill_holes_components_device(t.data_ptr(), dtype, zyx, mode, work.data_ptr(), s)
                t1 = time.perf_counter()
                st["components_ms"] = (t1 - t0) * 1e3
                if mode != "binary":
                    slots = 1 << 16
                    while slots < 4 * comps and slots < 1 << 30:
                        slots <<= 1
                    table, slots, edges = _grown_table(
                        t.device, slots, _native.fill_holes_table_workspace,
                        lambda table, slots: _native.fill_holes_graph_device(work.data_ptr(), zyx, table.data_ptr(), slots, s),
                        "fill holes: more touching component pairs (at most 2^30)")
                    t2 = time.perf_counter()
                    _native.fill_holes_enclose(work.data_ptr(), zyx, table.data_ptr(), slots, edges, s)
                    del table
                    t3 = time.perf_counter()
                    st.update(edges=edges, table_slots=slots, graph_ms=(t2 - t1) * 1e3, enclose_ms=(t3 - t2) * 1e3)
                    t1 = t3
                count = _native.fill_holes_apply_device(t.data_ptr(), dtype, zyx, work.data_ptr(), out.data_ptr(), s)
                st["apply_ms"] = (time.perf_counter() - t1) * 1e3
                del work
        if stats is not None:
            stats.update(st)
        res = DeviceChunk(out, voxel_offset=self.voxel_offset, voxel_size=self.voxel_size, layer_type=self.layer_type)
        return (res, count) if return_fill_count else res

    # ---- `skeletonize`: distance transform, geodesic field and TEASAR rounds on the device -----------------------------------
    def distance_transform(self, voxel_size=None) -> "DeviceChunk":
        """float32 distance of every voxel of a (z, y, x) segmentation to the nearest voxel of another id, outside the chunk
        counting as 0 (0 for id 0), in physical units (csrc/skeleton.cu; for integer voxel sizes bit-identical to
        scipy.ndimage.distance_transform_edt of each label's padded mask).  ``voxel_size`` is (z, y, x), the chunk's by default."""
        torch = _torch()
        t, code = self._ids("distance_transform")
        vs = self._physical_voxel_size(voxel_size)
        out = torch.empty(t.shape, dtype=torch.float32, device=t.device)
        with self._on_device():
            work = torch.empty(_native.edt_workspace(tuple(t.shape)), dtype=torch.uint8, device=t.device)
            _native.edt_device(t.data_ptr(), code, tuple(t.shape), vs, out.data_ptr(), work.data_ptr(), self._stream())
            del work
        return DeviceChunk(out, voxel_offset=self.voxel_offset, voxel_size=self.voxel_size)

    def skeletonize(self, voxel_size=None, scale: float = 4, const: float = 500, pdrf_scale: float = 100000, pdrf_exponent: int = 4,
                    dust_threshold: int = 1000, skip_ids=None, stats: Optional[dict] = None, fill_holes: bool = False) -> dict:
        """TEASAR skeletons of every object of a (z, y, x) segmentation (csrc/skeleton.cu, rules in
        oracle/skeleton_oracle.py; not kimimaro's skeletons): ``{id: Skeleton}`` in the chunk's own frame (vertices at voxel
        centres, x, y, z in physical units), ids ascending.  An object is a 26-connected component of one id; 0, the
        ``skip_ids`` and components of fewer than ``dust_threshold`` voxels are not skeletonized.  Same dtype and ndim checks as
        ``mesh``.  ``stats``, when given, receives the relaxation sweeps, rounds, paths and phase times of the call.
        ``fill_holes``: the objects are first filled with ``fill_holes("remove-enclosed")`` (kimimaro's fill_holes: labels that
        get filled in are deleted), so that a cavity does not make the skeleton loop around it."""
        from ..flow.skeleton import Skeleton, check_params
        torch = _torch()
        if fill_holes:
            self._ids("skeletonize")
            return self.fill_holes("remove-enclosed").skeletonize(voxel_size, scale, const, pdrf_scale, pdrf_exponent, dust_threshold,
                                                                  skip_ids, stats)
        t, code = self._ids("skeletonize")
        vs = self._physical_voxel_size(voxel_size)
        check_params(scale, const, pdrf_scale, pdrf_exponent, dust_threshold, vs, tuple(t.shape))
        skip = np.unique(selected_ids(skip_ids) if skip_ids is not None else np.zeros(0, np.uint64))
        zyx = tuple(t.shape)
        if min(zyx) == 0:
            return {}
        with self._on_device():
            d_skip = torch.from_numpy(skip.view(np.int64)).to(t.device) if skip.size else None
            work = torch.empty(_native.skeleton_workspace(zyx), dtype=torch.uint8, device=t.device)
            args = (t.data_ptr(), code, zyx, vs)
            counts = _native.skeleton_count_device(*args, d_skip.data_ptr() if d_skip is not None else 0, skip.size, int(dust_threshold),
                                                   work.data_ptr(), self._stream())
            buf = torch.empty(max(counts[2], 1), dtype=torch.uint8, device=t.device)
            n, st = _native.skeleton_device(*args, float(scale), float(const), float(pdrf_scale), int(pdrf_exponent), work.data_ptr(), counts,
                                            buf.data_ptr(), self._stream())
            out = _native.skeleton_read(buf.data_ptr(), zyx, vs, counts, n, self._stream())
            del buf, work
        if stats is not None:
            stats.update(st)
        return {k: Skeleton(*v) for k, v in out.items()}

    def __repr__(self):
        return f"DeviceChunk(shape={self.shape}, dtype={self.dtype}, voxel_offset={tuple(self.voxel_offset)}, device={self.tensor.device})"
