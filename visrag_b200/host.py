"""Host-side preparation of a batch (everything the reference does on the CPU before the GPU forward).

Mirrors, with the same results, the reference's
  * page slicing geometry   `modeling_minicpmv/modeling_minicpmv.py:482-592`  (slice_image & helpers),
  * placeholder text        `modeling_visrag_ret.py:57-84`, `modeling_minicpmv.py:247-274,595-609`,
  * tokenisation + image_bound `modeling_minicpmv.py:173-216`,
but produces *packed* (unpadded) sequences and uint8 slice tensors grouped by geometry, which is what the
H100 engine consumes. The geometry is split into a pure integer planner (`plan_slices`) — testable against
the reference's golden geometry without touching pixels — and the PIL resampling that executes a plan
(PIL's bicubic filter stays on the host because Recall parity depends on pixel-exact inputs, SURVEY.md H3).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import threading
import weakref
from collections import OrderedDict

import numpy as np

from .config import VisRAGConfig


def _snap(length: float, unit: int) -> int:
    """Nearest multiple of `unit`, at least one unit (reference ensure_divide, python round = banker's)."""
    return max(round(length / unit) * unit, unit)


def _fit(size: Tuple[float, float], target: int, unit: int, upscale: bool) -> Tuple[int, int]:
    """Size with (about) target^2 area, same aspect, sides snapped to `unit` (reference find_best_resize)."""
    w, h = size
    if w * h > target * target or upscale:
        r = w / h
        h = int(target / math.sqrt(r))
        w = int(h * r)
    return _snap(w, unit), _snap(h, unit)


@dataclass(frozen=True)
class SlicePlan:
    """How one page is cut: thumbnail size, grid (cols, rows) or None, refined full size, cell size."""
    source_size: Tuple[int, int]              # (w, h) of the thumbnail / only slice
    grid: Optional[Tuple[int, int]]           # (cols, rows); None when the page is not split
    refine_size: Optional[Tuple[int, int]]    # size the whole page is resized to before cropping cells
    cell_size: Optional[Tuple[int, int]]      # (w, h) of one crop

    @property
    def n_slices(self) -> int:
        return 1 if self.grid is None else 1 + self.grid[0] * self.grid[1]

    def slice_sizes(self) -> List[Tuple[int, int]]:
        return [self.source_size] + ([] if self.grid is None else [self.cell_size] * (self.grid[0] * self.grid[1]))


def plan_slices(width: int, height: int, cfg: VisRAGConfig) -> SlicePlan:
    """Integer geometry of `slice_image` for a (width x height) page."""
    S, P, cap = cfg.scale_resolution, cfg.patch_size, cfg.max_slice_nums
    parts = min(math.ceil(width * height / (S * S)), cap)
    if parts <= 1:
        return SlicePlan(_fit((width, height), S, P, True), None, None, None)
    aspect = math.log(width / height)
    best, best_err = (1, 1), float("inf")
    for n in (parts - 1, parts, parts + 1):
        if n == 1 or n > cap:
            continue
        for cols in range(1, n + 1):
            if n % cols:
                continue
            err = abs(aspect - math.log(cols / (n // cols)))
            if err < best_err:  # first minimum wins, same iteration order as the reference
                best, best_err = (cols, n // cols), err
    cols, rows = best
    cell = _fit((_snap(width, cols) / cols, _snap(height, rows) / rows), S, P, True)
    refine = (cell[0] * cols, cell[1] * rows)
    # split_to_patches uses int(refined / grid); identical to `cell` because refine is an exact multiple
    return SlicePlan(_fit((width, height), S, P, False), (cols, rows), refine, (int(refine[0] / cols), int(refine[1] / rows)))


def _rgb_array(image) -> np.ndarray:
    return np.asarray(image, dtype=np.uint8)


def render_slices(image, plan: SlicePlan) -> List[np.ndarray]:
    """Execute a plan with PIL bicubic resampling. Returns uint8 HWC arrays in LM order
    [thumbnail, row0col0, row0col1, ...] (`modeling_minicpmv.py:263-269`)."""
    from PIL import Image

    image = image.convert("RGB") if image.mode != "RGB" else image
    # PIL's resize to the identical size is a plain copy: skip it (same pixels)
    src = image if image.size == plan.source_size else image.resize(plan.source_size, Image.Resampling.BICUBIC)
    out = [_rgb_array(src)]
    if plan.grid is not None:
        refined = _rgb_array(image.resize(plan.refine_size, Image.Resampling.BICUBIC))
        cw, ch = plan.cell_size
        for i in range(plan.grid[1]):
            for j in range(plan.grid[0]):
                out.append(np.ascontiguousarray(refined[i * ch:(i + 1) * ch, j * cw:(j + 1) * cw]))
    return out


def placeholder_text(plan: Optional[SlicePlan], tokenizer, query_num: int) -> str:
    """`<image><unk>*64</image>` for the thumbnail, then `<slice>` rows `</slice>`; '' for text-only items."""
    if plan is None:
        return ""
    one = tokenizer.im_start + tokenizer.unk_token * query_num + tokenizer.im_end
    text = one
    if plan.grid is not None:
        cols, rows = plan.grid
        text += tokenizer.slice_start + "\n".join(one * cols for _ in range(rows)) + tokenizer.slice_end
    return text


_TOK_CACHE_MAX = 4096
_TOK_CACHES = weakref.WeakKeyDictionary()  # tokenizer object -> OrderedDict (LRU); dies with the tokenizer
_TOK_CACHES_LOCK = threading.Lock()


def _tok_cache(tokenizer):
    """The memo lives and dies with the tokenizer OBJECT (weak reference): `id()` values are reused after garbage
    collection, so a cache keyed on them could hand a new tokenizer another vocabulary's ids. Tokenizers that cannot be
    weakly referenced get no cache."""
    try:
        with _TOK_CACHES_LOCK:
            c = _TOK_CACHES.get(tokenizer)
            if c is None:
                c = _TOK_CACHES[tokenizer] = OrderedDict()
            return c
    except TypeError:
        return None


def tokenize(content: str, tokenizer, max_inp_length: Optional[int]) -> Tuple[np.ndarray, np.ndarray]:
    """ids (int32) truncated to max_inp_length and image_bound [n,2] = (index after <image>, index of </image>).
    Pure function of (tokenizer, content, max length): results are memoised per tokenizer object, LRU (every single-slice
    page shares one placeholder string, so a corpus batch tokenises it once)."""
    cache = _tok_cache(tokenizer)
    key = (content, max_inp_length)
    if cache is not None:
        with _TOK_CACHES_LOCK:
            hit = cache.get(key)
            if hit is not None:
                cache.move_to_end(key)
                return hit
    out = _tokenize(content, tokenizer, max_inp_length)
    if cache is not None:
        with _TOK_CACHES_LOCK:
            cache[key] = out
            if len(cache) > _TOK_CACHE_MAX:
                cache.popitem(last=False)
    return out


def _tokenize(content: str, tokenizer, max_inp_length: Optional[int]) -> Tuple[np.ndarray, np.ndarray]:
    ids = list(tokenizer.encode(content))
    if not tokenizer.add_bos_token:
        ids = [tokenizer.bos_id] + ids
    if max_inp_length is not None:
        ids = ids[:max_inp_length]
    ids = np.asarray(ids, dtype=np.int32)
    starts = np.flatnonzero(ids == tokenizer.im_start_id) + 1
    ends = np.flatnonzero(ids == tokenizer.im_end_id)
    n = max(len(starts), len(ends))
    if len(starts) != len(ends):
        raise ValueError("image span cut by max_inp_length: the reference cannot represent this either "
                         "(`modeling_minicpmv.py:179-193`); raise max_inp_length")
    bound = np.stack([starts[:n], ends[:n]], axis=1).astype(np.int32) if n else np.zeros((0, 2), np.int32)
    return ids, bound


MAX_DEVICE_PAGE_WIDTH = 12288  # vr_resample_u8 stages four source rows (up to 4 bytes per pixel) in shared memory


@dataclass
class PageJob:
    """A page whose slices the DEVICE front-end renders (frontend.DeviceFrontEnd): raw pixels + plan + where the
    results go (group key, index inside the group) for the thumbnail and for the first grid cell."""
    pixels: np.ndarray                                   # uint8 [H,W,3] (RGB) or [H,W,4] (Pillow's RGBX rows)
    plan: SlicePlan
    thumb: Optional[Tuple[Tuple[int, int], int]] = None
    cells: Optional[Tuple[Tuple[int, int], int]] = None


@dataclass
class PreparedBatch:
    """Packed representation of a batch of (text, image) items."""
    n_items: int
    seq_lens: np.ndarray                 # [B] int32
    cu_seqlens: np.ndarray               # [B+1] int32
    positions: np.ndarray                # [T] int32, position inside the sequence
    token_src: np.ndarray                # [T] int32: >=0 row of the vision buffer; <0 -> -(token_id+1)
    # (h,w) -> S slices: uint8 [h,w,3] arrays rendered on the host, or None = rendered on the device by one of `jobs`
    groups: Dict[Tuple[int, int], List[Optional[np.ndarray]]] = field(default_factory=dict)
    group_row0: Dict[Tuple[int, int], int] = field(default_factory=dict)      # (h,w) -> first slice index
    n_slices: int = 0
    jobs: List[PageJob] = field(default_factory=list)

    def pixel_bytes(self) -> int:
        """Pixel bytes that cross PCIe: host-rendered slices plus the raw pages of the device front-end."""
        return (sum(a.nbytes for lst in self.groups.values() for a in lst if a is not None)
                + sum(j.pixels.nbytes for j in self.jobs))


_POOL_WORKERS = 8
_pool_obj = None


def _pool():
    """Process-wide worker pool for per-page host work (created on first use; threads are daemonic helpers)."""
    global _pool_obj
    if _pool_obj is None:
        from concurrent.futures import ThreadPoolExecutor

        _pool_obj = ThreadPoolExecutor(max_workers=_POOL_WORKERS, thread_name_prefix="visrag-host")
    return _pool_obj


def prepare_batch(texts: Sequence[str], images: Sequence, tokenizer, cfg: VisRAGConfig,
                  max_inp_length: Optional[int] = 2048, device_frontend: bool = False) -> PreparedBatch:
    """Everything `VisRAG_Ret.forward` does before `get_vllm_embedding` (`modeling_visrag_ret.py:96-111`).
    With `device_frontend` the pages are not resampled here: their raw RGB pixels travel to the GPU and
    `frontend.DeviceFrontEnd` renders the same slices there (bit-identical to PIL)."""
    if len(texts) != len(images):
        raise ValueError("texts and images must have the same length")
    per_item_slices: list = []  # per item: list of host-rendered slices, or a PageJob
    ids_list, bound_list = [], []
    for text in texts:
        if not isinstance(text, str):
            raise NotImplementedError(f"chatml format expected, expect outmost type to be str but got {type(text)}")

    def one(item):
        text, image = item
        if image:
            plan = plan_slices(image.size[0], image.size[1], cfg)
            content = placeholder_text(plan, tokenizer, cfg.query_num) + "\n" + text
            # every page goes to the device as it is: Pillow's native RGBX rows when they can be exported zero-copy
            # (frontend.page_pixels), so the host neither resamples nor repacks pixels
            if device_frontend and image.size[0] <= MAX_DEVICE_PAGE_WIDTH:
                from .frontend import page_pixels

                return PageJob(page_pixels(image), plan), content
            return render_slices(image, plan), content
        return [], text

    n_img = sum(1 for im in images if im)
    items = list(zip(texts, images))
    # Threads only pay off when PIL resamples on the host (Image.resize releases the GIL; the reference uses
    # ThreadPoolExecutor(8) for the same reason). What is left with the device front-end - PIL's tobytes() behind
    # np.asarray - holds the GIL, so eight threads are no faster than one.
    if n_img >= 8 and not device_frontend:
        # one persistent pool and one task per worker: creating a pool and 128 futures per batch cost more than the work
        n_chunks = min(_POOL_WORKERS, len(items))
        bounds = [len(items) * i // n_chunks for i in range(n_chunks + 1)]
        parts = _pool().map(lambda ab: [one(it) for it in items[ab[0]:ab[1]]], zip(bounds, bounds[1:]))
        prepared = [r for part in parts for r in part]
    else:
        prepared = [one(it) for it in items]
    for (slices, content), image in zip(prepared, images):
        ids, bound = tokenize(content, tokenizer, max_inp_length)
        if isinstance(slices, PageJob) and len(bound) != slices.plan.n_slices:
            # truncated by max_inp_length (or stray markers): only some slices are consumed -> render on the host
            slices = render_slices(image, slices.plan)
        if isinstance(slices, PageJob):
            per_item_slices.append(slices)
            ids_list.append(ids)
            bound_list.append(bound)
            continue
        if len(bound) > len(slices):
            raise ValueError("more <image> spans in the text than slices")
        if any(int(e - s) != cfg.query_num for s, e in bound):
            raise ValueError("image span length != query_num (user text contains image markers?)")
        per_item_slices.append(slices[: len(bound)])
        ids_list.append(ids)
        bound_list.append(bound)

    # group slices by geometry; every slice gets a global index = position in the vision output buffer / query_num
    order: Dict[Tuple[int, int], List[Optional[np.ndarray]]] = {}
    slot: List[List[Tuple[Tuple[int, int], int]]] = []
    jobs: List[PageJob] = []
    for slices in per_item_slices:
        cur = []
        if isinstance(slices, PageJob):
            for n, (w, h) in enumerate(slices.plan.slice_sizes()):
                order.setdefault((h, w), []).append(None)
                cur.append(((h, w), len(order[(h, w)]) - 1))
            slices.thumb = cur[0]
            slices.cells = cur[1] if len(cur) > 1 else None
            jobs.append(slices)
        else:
            for s in slices:
                key = (s.shape[0], s.shape[1])
                order.setdefault(key, []).append(s)
                cur.append((key, len(order[key]) - 1))
        slot.append(cur)
    groups, row0, base = {}, {}, 0
    for key, lst in order.items():
        groups[key] = lst  # stacked straight into pinned staging memory by the engine (no intermediate copy)
        row0[key] = base
        base += len(lst)

    seq_lens = np.asarray([len(x) for x in ids_list], dtype=np.int32)
    cu = np.zeros(len(ids_list) + 1, dtype=np.int32)
    np.cumsum(seq_lens, out=cu[1:])
    T = int(cu[-1])
    positions = np.concatenate([np.arange(n, dtype=np.int32) for n in seq_lens]) if T else np.zeros(0, np.int32)
    src = np.empty(T, dtype=np.int32)
    for b, (ids, bound) in enumerate(zip(ids_list, bound_list)):
        seg = -(ids.astype(np.int64) + 1)
        for n, (s, e) in enumerate(bound):
            key, j = slot[b][n]
            seg[s:e] = (row0[key] + j) * cfg.query_num + np.arange(e - s)
        src[cu[b]:cu[b + 1]] = seg.astype(np.int32)
    return PreparedBatch(len(ids_list), seq_lens, cu, positions, src, groups, row0, base, jobs)


# ------------------------------------------------------------------------------------------------------------ prefix cache
# A text-only batch whose items all start with the same token prefix runs only the suffixes through the LM and reads the
# prefix's keys, values and residual rows from the engine's cache (encoder.VisRAGEngine, prefix_cache=True). Rows 0..P-1
# of a causal sequence depend only on tokens 0..P-1, so the cached rows are the rows the full run computes.
# A new entry needs at least this many shared tokens. tools/bench_prefix.py's sweep (full-size model, batches of 16 with
# 48-token suffixes, H100 80GB HBM3 at a 700 W power limit): the cached path is 1 % slower at P = 4, 5 % slower at 8 and
# 11 % faster at 16.
PREFIX_MIN_TOKENS = 16


def select_prefix(pb: PreparedBatch, cached: Sequence[Tuple[int, ...]],
                  min_tokens: Optional[int] = None) -> Optional[Tuple[Tuple[int, ...], bool]]:
    """The token-id prefix a batch runs from, and whether it is a new entry: (ids, new) or None for the full path.
    Only text-only batches qualify (page sequences share just BOS and <image>), and every item keeps at least one token
    of its own, so P <= P_max = min(seq_len) - 1. The longest entry of `cached` that starts every item and fits P_max wins;
    failing that, a batch of two or more items creates an entry from its items' longest common prefix (capped at P_max)
    when that has at least `min_tokens` (default PREFIX_MIN_TOKENS) tokens. Matching is on token ids, never on strings."""
    if pb.n_items == 0 or pb.n_slices or pb.jobs:
        return None
    p_max = int(pb.seq_lens.min()) - 1
    if p_max < 1:
        return None
    head = pb.token_src[pb.cu_seqlens[:-1, None] + np.arange(p_max)]
    if (head >= 0).any():  # a vision row: not a text-only batch
        return None
    head = -(head.astype(np.int64) + 1)  # [B, p_max] token ids
    best = None
    for ids in cached:
        n = len(ids)
        if 0 < n <= p_max and (best is None or n > len(best)) and np.array_equal(head[:, :n], np.broadcast_to(ids, (len(head), n))):
            best = tuple(ids)
    if best is not None:
        return best, False
    if pb.n_items < 2:
        return None
    differs = (head != head[0]).any(axis=0)
    n = int(np.argmax(differs)) if differs.any() else p_max
    if n < (PREFIX_MIN_TOKENS if min_tokens is None else min_tokens):
        return None
    return tuple(int(i) for i in head[0, :n]), True


def suffix_batch(pb: PreparedBatch, prefix_len: int) -> PreparedBatch:
    """The batch without the first `prefix_len` tokens of every item. Positions stay absolute (prefix_len + i), as RoPE
    needs them; seq_lens / cu_seqlens count the suffix tokens only."""
    keep = pb.positions >= prefix_len
    B = pb.n_items
    cu = pb.cu_seqlens - prefix_len * np.arange(B + 1, dtype=np.int32)
    return PreparedBatch(B, pb.seq_lens - prefix_len, cu.astype(np.int32), pb.positions[keep], pb.token_src[keep])
