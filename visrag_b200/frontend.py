"""Device image front-end (SURVEY.md §8f.2): page slicing + PIL-bit-compatible bicubic resampling on the GPU.

The reference resizes every page on the host with `PIL.Image.resize(size, Image.BICUBIC)`
(`modeling_minicpmv/modeling_minicpmv.py:509,519,531` inside `slice_image`) and crops the grid cells with
`split_to_patches` (`:571-592`). Retrieval parity depends on pixel-exact inputs, so the device path reproduces
Pillow's 8-bit resampler exactly (Pillow `src/libImaging/Resample.c`, `ImagingResample` with the bicubic filter —
a third-party dependency of the reference, pinned `Pillow==10.1.0` in its requirements; the algorithm is unchanged in
the Pillow 12 installed here, which the tests compare against bit for bit):

  * per axis, `precompute_coeffs`: scale = in/out, filterscale = max(scale, 1), support = 2*filterscale,
    ksize = ceil(support)*2+1; for output index i: center = (i+0.5)*scale, window [xmin, xmin+n) =
    [int(center-support+0.5) clipped at 0, int(center+support+0.5) clipped at in), weights
    bicubic((x+xmin-center+0.5)/filterscale) (a = -0.5) normalised by their sum — all in IEEE double;
  * `normalize_coeffs_8bpc`: fixed point with 22 fractional bits, round half away from zero;
  * horizontal pass first (only over the source rows the vertical pass needs), 8-bit intermediate with
    `clip8((1<<21 + sum(pixel*k)) >> 22)`, then the vertical pass; a pass whose size does not change is skipped.

The coefficient tables are computed here on the host (tiny, cached per (in,out) pair) and the two passes run as CUDA
kernels behind `vr_resample_u8` (csrc/resample.cu). The kernels write straight into the engine's per-geometry slice
buffers (cell layout), so the grid crop costs nothing.
"""
from __future__ import annotations

import math
from functools import lru_cache
from typing import Tuple

import numpy as np

PRECISION_BITS = 32 - 8 - 2


def _bicubic(x: float) -> float:
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


@lru_cache(maxsize=512)
def resample_coeffs(in_size: int, out_size: int) -> Tuple[int, np.ndarray, np.ndarray]:
    """Pillow `precompute_coeffs` + `normalize_coeffs_8bpc` for the full-axis box (0, in_size), bicubic.
    Returns (ksize, bounds int32 [out,2] = (first source index, tap count), coeffs int32 [out, ksize])."""
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), dtype=np.int32)
    kk = np.zeros((out_size, ksize), dtype=np.int32)
    ss = 1.0 / filterscale
    one = float(1 << PRECISION_BITS)
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [_bicubic((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for v in w:
            ww += v
        for x in range(xmax):
            v = w[x] / ww if ww != 0.0 else w[x]
            kk[xx, x] = int(-0.5 + v * one) if v < 0 else int(0.5 + v * one)
        bounds[xx] = (xmin, xmax)
    return ksize, bounds, kk


class DeviceFrontEnd:
    """Runs slice plans on the GPU for stacks of equal-sized pages. Coefficient tables live on the device, cached per
    (in, out) axis pair. All launches go to the current CUDA stream."""

    def __init__(self, device):
        self.device = device
        self._tables = {}

    def _axis(self, n_in: int, n_out: int, tap_major: bool):
        """-> (ksize, bounds_dev, coeffs_dev, first_row, row_count) or None when the axis keeps its size.
        `tap_major`: coefficients as [ksize, out] (the horizontal pass reads them coalesced) instead of [out, ksize]."""
        import torch

        if n_in == n_out:
            return None
        key = (n_in, n_out, tap_major)
        if key not in self._tables:
            ksize, bounds, kk = resample_coeffs(n_in, n_out)
            first = int(bounds[0, 0])
            last = int(bounds[-1, 0] + bounds[-1, 1])
            if tap_major:
                kk = np.ascontiguousarray(kk.T)
            self._tables[key] = (ksize, torch.from_numpy(bounds).to(self.device), torch.from_numpy(kk).to(self.device),
                                 first, last - first)
        return self._tables[key]

    def resize_into(self, pages, out_w: int, out_h: int, out, first_cell, cell_w: int, cell_h: int) -> None:
        """pages uint8 [n,H,W,3] or [n,H,W,4] (RGBX, Pillow's native rows) on the device -> bicubic (out_h x out_w), cut
        into cell_h x cell_w cells which are written to `out` [*, cell_h, cell_w, 3] starting at slice first_cell[i] for
        page i (`first_cell` int32 [n], device)."""
        from . import _lib as L

        n, H, W, ps = pages.shape
        L.check_device(pages)  # the engine's upload() enters its own device before calling this
        h = self._axis(W, out_w, True)
        v = self._axis(H, out_h, False)
        tmp = None
        r0, rc = (v[3], v[4]) if v is not None else (0, H)
        if h is not None and v is not None:
            import torch

            tmp = torch.empty((n, rc, (out_w * 3 + 3) & ~3), dtype=torch.uint8, device=pages.device)  # 4-byte row pitch
        L.check(L.lib().vr_resample_u8(
            pages.data_ptr(), ps, n, H, W,
            h[1].data_ptr() if h else None, h[2].data_ptr() if h else None, h[0] if h else 0,
            v[1].data_ptr() if v else None, v[2].data_ptr() if v else None, v[0] if v else 0,
            r0, rc, out_h, out_w, tmp.data_ptr() if tmp is not None else None, out.data_ptr(), first_cell.data_ptr(),
            cell_h, cell_w, L.stream_ptr()))


def page_pixels(image) -> np.ndarray:
    """uint8 pixels of a PIL RGB image for the device front-end, WITHOUT repacking when possible: Pillow stores mode "RGB"
    as RGBX rows (4 bytes per pixel) and exports that buffer zero-copy through the Arrow C data interface (Pillow >= 11.2),
    so the page can be copied straight into pinned memory as [H, W, 4]; `np.asarray(image)` instead goes through
    `tobytes()`, which repacks to RGB under the GIL. Falls back to that ([H, W, 3]) when the
    export is unavailable (older Pillow, no pyarrow, images stored in several blocks)."""
    if image.mode != "RGB":
        image = image.convert("RGB")
    try:
        import pyarrow as pa

        flat = pa.array(image).flatten().to_numpy(zero_copy_only=True)
        w, h = image.size
        if flat.dtype == np.uint8 and flat.size == w * h * 4:
            return flat.reshape(h, w, 4)  # keeps the Arrow array (and through it the image buffer) alive
    except Exception:  # noqa: BLE001 - any failure of the optional fast path means: use the portable one
        pass
    return np.ascontiguousarray(np.asarray(image, dtype=np.uint8))
