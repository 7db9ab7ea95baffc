"""Search a database of scenes on the device (csrc/search.cu; DESIGN.md, "Scene search contract").

OpenScene's per-voxel features answer open-vocabulary queries over many scenes at once: rare-object search by name (CLIP
text rows) and image-based retrieval (CLIP image rows).  ``SceneIndex`` keeps the operand rows of many scenes in one
fixed device arena, and ``query`` scores every row against the queries on the tensor cores, with the bits
``osb_match_scores`` gives the same row, and returns

- the k best rows per query over the whole index (score, scene, row within the scene);
- per scene and query the best score and its row, and optionally how many rows score at or above a threshold.

The [N, nq] scores never exist in memory.  One memset and two launches serve up to 96 queries, and each such slice reads
the index once; more queries run slice after slice.  Nothing synchronises the host.

An index built with ``coords=True`` also keeps each row's voxel coordinates, and ``regions`` groups each query's hits
(rows at or above a threshold) into spatially connected regions on the device (csrc/regions.cu; DESIGN.md, "Region
contract"): the objects a search for a name or an image is after, with their boxes, sizes and best hits.

An index built with ``storage='fp8'`` keeps each row as e4m3 codes and one power-of-two exponent (C + 1 bytes instead of
2 C; DESIGN.md, "FP8 index contract"): twice the rows in the same memory, and each query slice reads half the bytes.  It
answers exactly what an fp16 index holding the dequantized rows answers.
"""
from collections import namedtuple

import torch

from . import _cabi as C

MAX_QUERIES = 96      # OSB_SEARCH_MAX_QUERIES: one 96-column wgmma pass per launch
MAX_K = 32            # OSB_SEARCH_MAX_K
MAX_REGIONS = 32      # OSB_REGIONS_MAX_R
C_ST_COUNT, C_ST_RANGE, C_ST_DUP = 1, 2, 4      # OSB_REGIONS_ST_*: the status word of osb_search_hits / osb_regions

SearchResult = namedtuple('SearchResult', 'score scene row scene_max scene_argmax scene_count')
SearchResult.__doc__ = """score fp16 / scene int64 / row int64 [nq, k]: best first, (-inf, -1, -1) past the last non-NaN row;
scene_max fp16 / scene_argmax int64 [S, nq]: (-inf, -1) for a scene without a non-NaN score; scene_count int64 [S, nq]
(rows with float(score) >= threshold[q]) or None."""

RegionResult = namedtuple('RegionResult', 'score scene row size box_min box_max n_regions '
                                          'hit_query hit_scene hit_row hit_score hit_region')
RegionResult.__doc__ = """score fp16 / scene int64 / row int64 / size int64 [nq, R], box_min / box_max int32 [nq, R, 3]: the
best regions per query, ranked by the search key of their best hit (score, scene and row within the scene of that hit);
unused slots (-inf, -1, -1, 0, 0, 0).  n_regions int64 [S, nq]: regions of at least min_voxels voxels.  With hits=True,
hit_query / hit_scene / hit_row int64, hit_score fp16 and hit_region int64 [n_hits] list every hit sorted by (query,
global row), hit_region the rank of its region in its query's list or -1; otherwise None."""


class SceneIndex:
    """A fixed device arena of fp16 operand rows [capacity_rows, channels], filled scene after scene by ``add``.

    Scene ids follow the order of ``add``.  The arena never grows and is never re-copied.  With ``coords=True`` an int32
    [capacity_rows, 4] arena holds each row's voxel coordinates (x, y, z, 0), which ``regions`` needs.

    ``storage='fp8'`` stores each row as e4m3 codes (``codes``, uint8 [capacity_rows, channels]) and an int8 exponent
    (``row_exp``, [capacity_rows]) instead of ``rows``: the row it stands for is d = code * 2^e, an exact fp16 row, and
    every result is the one an fp16 index holding d gives.  C + 5 bytes per row with the scene id, against 2 C + 4."""

    def __init__(self, capacity_rows, channels=768, device=None, coords=False, storage='fp16'):
        if storage not in ('fp16', 'fp8'):
            raise ValueError(f"SceneIndex: storage must be 'fp16' or 'fp8' (got {storage!r})")
        if channels not in (512, 768):
            raise ValueError(f"SceneIndex: channels must be 512 or 768 (got {channels})")
        if not 1 <= capacity_rows < 2 ** 31:
            raise ValueError(f"SceneIndex: capacity_rows must lie in 1..2^31-1 (got {capacity_rows})")
        self.device = torch.device(device if device is not None else 'cuda', )
        if self.device.type != 'cuda':
            raise RuntimeError("openscene_b200: SceneIndex lives on a CUDA device; there is no CPU fallback for this path")
        if self.device.index is None:
            self.device = torch.device('cuda', torch.cuda.current_device())
        self.capacity = int(capacity_rows)
        self.channels = int(channels)
        self.storage = storage
        if storage == 'fp16':
            self.rows = torch.empty((self.capacity, self.channels), dtype=torch.float16, device=self.device)
            self.codes = self.row_exp = None
        else:
            self.rows = None
            self.codes = torch.empty((self.capacity, self.channels), dtype=torch.uint8, device=self.device)
            self.row_exp = torch.empty(self.capacity, dtype=torch.int8, device=self.device)
        self.row_scene = torch.empty(self.capacity, dtype=torch.int32, device=self.device)
        self.coords = torch.zeros((self.capacity, 4), dtype=torch.int32, device=self.device) if coords else None
        self._off = [0]                                    # host offsets, n_scenes + 1
        self._off_dev = torch.zeros(64, dtype=torch.int64, device=self.device)
        self.names = []

    @property
    def n_rows(self):
        return self._off[-1]

    @property
    def n_scenes(self):
        return len(self._off) - 1

    def scene_rows(self, scene):
        """The rows [n, C] of one scene: a view into the arena, or on an FP8 index a new fp16 tensor of the dequantized
        rows d = code * 2^e (exact; NaN rows stay NaN)."""
        a, b = self._off[scene], self._off[scene + 1]
        if self.codes is None:
            return self.rows[a:b]
        scale = ((self.row_exp[a:b].int() + 127) << 23).view(torch.float32)       # 2^e, exactly
        return (self.codes[a:b].view(torch.float8_e4m3fn).float() * scale[:, None]).half()

    def _operand(self):
        """the entry-point suffix and the row arguments of the storage"""
        if self.codes is None:
            return '', [C.ptr(self.rows)]
        return '_f8', [C.ptr(self.codes), C.ptr(self.row_exp)]

    def scene_coords(self, scene):
        """The voxel coordinates [n, 4] (x, y, z, 0) of one scene, row for row with ``scene_rows`` (a view)."""
        if self.coords is None:
            raise RuntimeError("SceneIndex.scene_coords: the index was built without coordinates (coords=True)")
        return self.coords[self._off[scene]:self._off[scene + 1]]

    def add(self, rows, name=None, coords=None):
        """Append one scene's operand rows (fp16 [n, C]; fp32 is taken as ``.half()``, the 'distill' operand) and return
        its scene id.  ``coords``: integer voxel coordinates [n, 3], or [n, 4] in MinkowskiEngine's (batch, x, y, z)
        layout whose batch column is dropped, row for row with ``rows``; required on an index built with coordinates and
        refused on one without.  An empty scene, a wrong width, dtype or device, or a full arena is refused before
        anything is copied.  An FP8 index quantizes the rows on the device (``osb_index_quantize_f8``, one launch)."""
        if not isinstance(rows, torch.Tensor) or rows.dim() != 2:
            raise ValueError("SceneIndex.add: rows must be a 2-D tensor [n, C]")
        if rows.dtype not in (torch.float16, torch.float32):
            raise TypeError(f"SceneIndex.add: rows must be fp16 or fp32 (got {rows.dtype})")
        if rows.device != self.device:
            raise ValueError(f"SceneIndex.add: rows are on {rows.device}, the index on {self.device}")
        n, c = rows.shape
        if c != self.channels:
            raise ValueError(f"SceneIndex.add: rows have width {c}, the index {self.channels}")
        if n < 1:
            raise ValueError("SceneIndex.add: empty scene")
        if self.coords is None and coords is not None:
            raise ValueError("SceneIndex.add: coordinates given to an index built without them (coords=True)")
        if self.coords is not None:
            if coords is None:
                raise ValueError("SceneIndex.add: this index keeps coordinates; pass coords [n, 3] or [n, 4]")
            if not isinstance(coords, torch.Tensor) or coords.dim() != 2 or coords.shape[1] not in (3, 4):
                raise ValueError("SceneIndex.add: coords must be a 2-D tensor [n, 3] (x, y, z) or [n, 4] (batch, x, y, z)")
            if coords.dtype not in (torch.int32, torch.int64, torch.int16, torch.uint8, torch.int8):
                raise TypeError(f"SceneIndex.add: coords must be integer (got {coords.dtype})")
            if coords.shape[0] != n:
                raise ValueError(f"SceneIndex.add: {coords.shape[0]} coordinates for {n} rows")
            if coords.device != self.device:
                raise ValueError(f"SceneIndex.add: coords are on {coords.device}, the index on {self.device}")
        o = self.n_rows
        if o + n > self.capacity:
            raise RuntimeError(f"SceneIndex.add: {n} rows do not fit ({self.capacity - o} of {self.capacity} left)")
        s = self.n_scenes
        if self.codes is None:
            self.rows[o:o + n].copy_(rows)                # fp32 -> fp16 rounds to nearest even, as `.half()`
        else:
            src = rows.contiguous()
            if src.data_ptr() % 16:
                src = src.clone()
            with torch.cuda.device(self.device):
                C.call('osb_index_quantize_f8', C.ptr(src), int(src.dtype == torch.float16), n, self.channels,
                       C.ptr(self.codes[o:o + n]), C.ptr(self.row_exp[o:o + n]), C.stream_ptr())
        self.row_scene[o:o + n].fill_(s)
        if self.coords is not None:
            self.coords[o:o + n, :3].copy_(coords[:, -3:])
        if s + 2 > self._off_dev.numel():
            grown = torch.zeros(2 * self._off_dev.numel(), dtype=torch.int64, device=self.device)
            grown[:self._off_dev.numel()].copy_(self._off_dev)
            self._off_dev = grown
        self._off_dev[s + 1:s + 2].fill_(o + n)           # a fill kernel, not a copy from host memory
        self._off.append(o + n)
        self.names.append(name)
        return s

    def query(self, queries, k=1, threshold=None):
        """Score queries (fp16/fp32 [nq, C] or [C]) against every row.  ``threshold`` (float or [nq]) turns on the
        per-scene counts.  Any nq >= 1: one launch pair per slice of 96 queries, each slice reading the index once.
        Returns a ``SearchResult`` of device tensors."""
        if self.n_scenes == 0:
            raise RuntimeError("SceneIndex.query: the index is empty")
        if not 1 <= k <= MAX_K:
            raise ValueError(f"SceneIndex.query: k={k} outside 1..{MAX_K}")
        q = queries.to(device=self.device, dtype=torch.float16)
        if q.dim() == 1:
            q = q.unsqueeze(0)
        if q.dim() != 2 or q.shape[1] != self.channels or q.shape[0] < 1:
            raise ValueError(f"SceneIndex.query: queries must be [nq >= 1, {self.channels}] (got {tuple(queries.shape)})")
        nq = q.shape[0]
        thr = None
        if threshold is not None:
            if isinstance(threshold, torch.Tensor):
                thr = threshold.to(device=self.device, dtype=torch.float32).reshape(-1)
            else:     # a number or a list: filled on the device, no copy that would wait for the host
                vals = [float(threshold)] if isinstance(threshold, (int, float)) else [float(v) for v in threshold]
                thr = torch.empty(len(vals), dtype=torch.float32, device=self.device)
                for i, v in enumerate(vals) if len(vals) > 1 else ():
                    thr[i] = v
                if len(vals) == 1:
                    thr.fill_(vals[0])
            if thr.numel() == 1:
                thr = thr.expand(nq)
            if thr.numel() != nq:
                raise ValueError(f"SceneIndex.query: {thr.numel()} thresholds for {nq} queries")
            thr = thr.contiguous()
        parts = [self._query(q[i:i + MAX_QUERIES].contiguous(), k, None if thr is None else thr[i:i + MAX_QUERIES])
                 for i in range(0, nq, MAX_QUERIES)]
        if len(parts) == 1:
            return parts[0]
        return SearchResult(*(None if parts[0][j] is None else torch.cat([p[j] for p in parts], dim=0 if j < 3 else 1)
                              for j in range(6)))

    def _queries(self, queries, what):
        q = queries.to(device=self.device, dtype=torch.float16)
        if q.dim() == 1:
            q = q.unsqueeze(0)
        if q.dim() != 2 or q.shape[1] != self.channels or q.shape[0] < 1:
            raise ValueError(f"SceneIndex.{what}: queries must be [nq >= 1, {self.channels}] (got {tuple(queries.shape)})")
        return q

    def _thresholds(self, threshold, nq, what):
        if isinstance(threshold, torch.Tensor):
            thr = threshold.to(device=self.device, dtype=torch.float32).reshape(-1)
        else:     # a number or a list: filled on the device, no copy that would wait for the host
            vals = [float(threshold)] if isinstance(threshold, (int, float)) else [float(v) for v in threshold]
            thr = torch.empty(len(vals), dtype=torch.float32, device=self.device)
            if len(vals) == 1:
                thr.fill_(vals[0])
            else:
                for i, v in enumerate(vals):
                    thr[i] = v
        if thr.numel() == 1:
            thr = thr.expand(nq)
        if thr.numel() != nq:
            raise ValueError(f"SceneIndex.{what}: {thr.numel()} thresholds for {nq} queries")
        return thr.contiguous()

    def regions(self, queries, threshold, max_regions=8, reach=1, min_voxels=1, hits=False, max_hits=2 ** 26):
        """Group each query's hits, the rows r with float(s[r, q]) >= threshold[q] (s the bits ``query`` scores), into
        connected regions: two hits of one scene are adjacent when their coordinates differ by at most ``reach`` (1 or
        2) on every axis.  Returns a ``RegionResult`` with the ``max_regions`` (1..32) best regions of at least
        ``min_voxels`` voxels per query.  Any nq: slices of 96 queries.

        Two host synchronisations: one read of the total hit count (from ``osb_search``'s counts), which sizes the hit
        buffers and is refused above ``max_hits`` before they are allocated, and one read of a status word at the end,
        which raises when a hit's coordinate lies outside |x|, |y|, |z| < 2^17 - 256 or two hits of one (scene, query)
        share a voxel.  Duplicate coordinates among rows that are not hits are not inspected."""
        if self.coords is None:
            raise RuntimeError("SceneIndex.regions: the index was built without coordinates (coords=True)")
        if self.n_scenes == 0:
            raise RuntimeError("SceneIndex.regions: the index is empty")
        if not 1 <= max_regions <= MAX_REGIONS:
            raise ValueError(f"SceneIndex.regions: max_regions={max_regions} outside 1..{MAX_REGIONS}")
        if reach not in (1, 2):
            raise ValueError(f"SceneIndex.regions: reach={reach} outside 1..2")
        if min_voxels < 1:
            raise ValueError(f"SceneIndex.regions: min_voxels={min_voxels} below 1")
        q = self._queries(queries, 'regions')
        nq, S, dev, R = q.shape[0], self.n_scenes, self.device, int(max_regions)
        thr = self._thresholds(threshold, nq, 'regions')
        slices = [(i, q[i:i + MAX_QUERIES].contiguous(), thr[i:i + MAX_QUERIES].contiguous())
                  for i in range(0, nq, MAX_QUERIES)]
        counts = [self._query(qs, 1, ts).scene_count for _, qs, ts in slices]
        with torch.cuda.device(dev):
            totals = [int(t) for t in torch.stack([c.sum() for c in counts]).tolist()]      # host sync 1
        total = sum(totals)
        if total > max_hits:
            raise RuntimeError(f"SceneIndex.regions: {total} hits exceed max_hits={max_hits}; raise the threshold or "
                               f"max_hits")
        off_host = (C.I64 * (S + 1))(*self._off)
        parts = []
        with torch.cuda.device(dev):
            status = torch.zeros(1, dtype=torch.int32, device=dev)
            for (q0, qs, ts), cnt, h in zip(slices, counts, totals):
                m = qs.shape[0]
                if qs.data_ptr() % 16:
                    qs = qs.clone()
                key = torch.empty(h, dtype=torch.int64, device=dev)
                hsc = torch.empty(h, dtype=torch.float16, device=dev)
                if h:
                    ws_bytes = C.lib().osb_search_hits_workspace_bytes(S, m, h)
                    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
                    sfx, operand = self._operand()
                    C.call('osb_search_hits' + sfx, *operand, C.ptr(self.row_scene), self.n_rows, self.channels,
                           off_host, S, C.ptr(qs), m, C.ptr(ts), C.ptr(cnt), h, C.ptr(key), C.ptr(hsc), C.ptr(status),
                           C.ptr(ws), ws_bytes, C.stream_ptr())
                    del ws
                out = [torch.empty((m, R), dtype=torch.float16, device=dev)] + \
                      [torch.empty((m, R), dtype=torch.int64, device=dev) for _ in range(3)] + \
                      [torch.empty((m, R, 3), dtype=torch.int32, device=dev) for _ in range(2)] + \
                      [torch.empty((S, m), dtype=torch.int64, device=dev)]
                hit_out = [torch.empty(h, dtype=torch.int64, device=dev) for _ in range(4)] if hits else [None] * 4
                ws_bytes = C.lib().osb_regions_workspace_bytes(h)
                ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev) if h else None
                C.call('osb_regions', C.ptr(key), C.ptr(hsc), h, C.ptr(self.coords), C.ptr(self.row_scene),
                       C.ptr(self._off_dev), self.n_rows, S, m, R, int(reach), int(min_voxels), *[C.ptr(t) for t in out],
                       *[C.ptr(t) for t in hit_out], C.ptr(status), C.ptr(ws), ws_bytes, C.stream_ptr())
                del ws
                if hits:
                    hit_out[0] += q0
                    parts.append(out + [hit_out[0], hit_out[1], hit_out[2], hsc, hit_out[3]])
                else:
                    parts.append(out + [None] * 5)
            st = int(status.item())                                                         # host sync 2
        if st & C_ST_RANGE:
            raise RuntimeError("SceneIndex.regions: a hit's coordinate lies outside |x|, |y|, |z| < 2^17 - 256")
        if st & C_ST_DUP:
            raise RuntimeError("SceneIndex.regions: two hits of one (scene, query) share a voxel (duplicate coordinates)")
        if st:
            raise RuntimeError(f"SceneIndex.regions: the hit list does not match the search's counts (status {st})")
        if len(parts) == 1:
            return RegionResult(*parts[0])
        cat = lambda j, d: None if parts[0][j] is None else torch.cat([p[j] for p in parts], dim=d)
        return RegionResult(*[cat(j, 1 if j == 6 else 0) for j in range(12)])

    def _query(self, q, k, thr):
        nq, S, dev = q.shape[0], self.n_scenes, self.device
        if q.data_ptr() % 16:
            q = q.clone()
        with torch.cuda.device(dev):
            score = torch.empty((nq, k), dtype=torch.float16, device=dev)
            scene = torch.empty((nq, k), dtype=torch.int64, device=dev)
            row = torch.empty((nq, k), dtype=torch.int64, device=dev)
            smax = torch.empty((S, nq), dtype=torch.float16, device=dev)
            sarg = torch.empty((S, nq), dtype=torch.int64, device=dev)
            cnt = torch.empty((S, nq), dtype=torch.int64, device=dev) if thr is not None else None
            ws_bytes = C.lib().osb_search_workspace_bytes(S, nq, k)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
            off_host = (C.I64 * (S + 1))(*self._off)
            sfx, operand = self._operand()
            C.call('osb_search' + sfx, *operand, C.ptr(self.row_scene), self.n_rows, self.channels, off_host,
                   C.ptr(self._off_dev), S, C.ptr(q), nq, k, C.ptr(thr), C.ptr(score), C.ptr(scene), C.ptr(row),
                   C.ptr(smax), C.ptr(sarg), C.ptr(cnt), C.ptr(ws), ws_bytes, C.stream_ptr())
        return SearchResult(score, scene, row, smax, sarg, cnt)


def regions_hit_bytes(n_hits, n_scenes, nq, hits=False):
    """Device bytes a ``regions`` slice of nq queries holds at its peak for n_hits hits: the sorted hit list (10 B per
    hit), the larger of the two workspaces, and the per-hit outputs (34 B per hit) when hits=True."""
    if n_hits == 0:
        return 0
    ws = max(C.lib().osb_search_hits_workspace_bytes(n_scenes, nq, n_hits), C.lib().osb_regions_workspace_bytes(n_hits))
    return 10 * n_hits + int(ws) + (32 * n_hits if hits else 0)


def search_workspace_bytes(n_scenes, nq, k):
    """Device workspace of one launch pair (independent of the number of rows)."""
    return int(C.lib().osb_search_workspace_bytes(n_scenes, nq, k))
