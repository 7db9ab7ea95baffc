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

``label`` labels every row against a vocabulary, as OpenScene segments a scene (the argmax over the label set), and keeps
the labels current through later adds (csrc/label.cu; DESIGN.md, "Label contract"): ``labels`` gives a scene's
segmentation, ``class_counts`` the rows of each class per scene, and ``class_regions`` the connected pieces of each
class (zero-shot instance proposals) through the same region grower as ``regions``.

``ShardedSceneIndex`` spreads one database over the ranks of a process group (csrc/shard.cu; DESIGN.md, "Sharded index
contract"): each rank keeps the scenes it computed, a query runs ``k_search`` on every shard, and the small per-shard
results are merged on the device after one collective.  Every output is bit for bit the output of one ``SceneIndex``
that adds the scenes in ascending global id.
"""
import bisect
import operator
from collections import namedtuple

import torch

from . import _cabi as C

MAX_QUERIES = 96      # OSB_SEARCH_MAX_QUERIES: one 96-column wgmma pass per launch
MAX_K = 32            # OSB_SEARCH_MAX_K
MAX_REGIONS = 32      # OSB_REGIONS_MAX_R
MAX_VOCAB = 1 << 20   # OSB_MATCH_TOPK_MAX_TEXT
MAX_COUNTS = 1 << 27  # OSB_LABEL_MAX_COUNTS
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
        self.vocab = self.row_label = self.row_label_score = None       # set by label()

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
        if self.vocab is not None:
            self._label_rows(o, o + n)
        self._off.append(o + n)
        self.names.append(name)
        return s

    # ------------------------------------------------------------------ labels (DESIGN.md, "Label contract")
    def label(self, vocab):
        """Label every row against a vocabulary (fp16 / fp32 [K, C], 1 <= K <= 2^20; fp32 is taken as ``.half()``): the
        label of row r is column 0 of ``osb_match_topk(topk=1)`` on the row, the first NaN else the first maximum with
        -0 == +0, which on NaN-free rows is ``evaluate.py``'s ``torch.max(pred, 1)[1]``; its fp16 score is kept with it.
        An FP8 index labels the rows d it stands for (``osb_match_topk_f8``).  The first call allocates ``row_label``
        (int64) and ``row_label_score`` (fp16) over the capacity, 10 B per row.  The index keeps a copy of the
        vocabulary, and every later ``add`` labels its scene in the same call, so every row always carries its label
        under the current vocabulary; calling ``label`` again replaces the vocabulary and every label.  One launch, no
        host synchronisation; on an empty index only the vocabulary is stored."""
        if not isinstance(vocab, torch.Tensor) or vocab.dim() != 2:
            raise ValueError("SceneIndex.label: vocab must be a 2-D tensor [K, C]")
        if vocab.dtype not in (torch.float16, torch.float32):
            raise TypeError(f"SceneIndex.label: vocab must be fp16 or fp32 (got {vocab.dtype})")
        if vocab.device != self.device:
            raise ValueError(f"SceneIndex.label: vocab is on {vocab.device}, the index on {self.device}")
        K, c = vocab.shape
        if c != self.channels:
            raise ValueError(f"SceneIndex.label: vocab has width {c}, the index {self.channels}")
        if not 1 <= K <= MAX_VOCAB:
            raise ValueError(f"SceneIndex.label: {K} classes outside 1..{MAX_VOCAB}")
        with torch.cuda.device(self.device):
            self.vocab = vocab.to(torch.float16, copy=True).contiguous()
            if self.row_label is None:
                self.row_label = torch.empty(self.capacity, dtype=torch.int64, device=self.device)
                self.row_label_score = torch.empty(self.capacity, dtype=torch.float16, device=self.device)
        if self.n_rows:
            self._label_rows(0, self.n_rows)

    def _label_rows(self, a, b):
        K = self.vocab.shape[0]
        with torch.cuda.device(self.device):
            if self.codes is None:
                C.call('osb_match_topk', C.ptr(self.rows[a:b]), 1, b - a, self.channels, None, b - a, C.ptr(self.vocab),
                       K, 0, 1, C.ptr(self.row_label_score[a:b]), C.ptr(self.row_label[a:b]), None, C.stream_ptr())
            else:
                C.call('osb_match_topk_f8', C.ptr(self.codes[a:b]), C.ptr(self.row_exp[a:b]), b - a, self.channels,
                       C.ptr(self.vocab), K, 1, C.ptr(self.row_label_score[a:b]), C.ptr(self.row_label[a:b]), None,
                       C.stream_ptr())

    def _labelled(self, what):
        if self.vocab is None:
            raise RuntimeError(f"SceneIndex.{what}: the index is not labelled; call label(vocab) first")
        return self.vocab.shape[0]

    def labels(self, scene):
        """The labels (int64 [n]) and label scores (fp16 [n]) of one scene, row for row with ``scene_rows`` (views)."""
        self._labelled('labels')
        a, b = self._off[scene], self._off[scene + 1]
        return self.row_label[a:b], self.row_label_score[a:b]

    def _classes(self, classes, K, what):
        """a host sequence of distinct class ids in [0, K) -> list of ints (refused before any launch)"""
        if isinstance(classes, torch.Tensor):
            if classes.device.type != 'cpu' or classes.dim() != 1 or classes.dtype.is_floating_point or \
                    classes.dtype == torch.bool:
                raise ValueError(f"SceneIndex.{what}: classes must be a 1-D integer CPU tensor or a host sequence")
            ids = [int(v) for v in classes.tolist()]
        else:
            if isinstance(classes, (str, bytes)) or not hasattr(classes, '__iter__'):
                raise ValueError(f"SceneIndex.{what}: classes must be a sequence of class ids")
            ids = []
            for v in classes:
                if isinstance(v, bool):
                    raise ValueError(f"SceneIndex.{what}: class ids must be integers (got {v!r})")
                try:
                    ids.append(operator.index(v))
                except TypeError:
                    raise ValueError(f"SceneIndex.{what}: class ids must be integers (got {v!r})")
        if not ids:
            raise ValueError(f"SceneIndex.{what}: no classes")
        bad = [v for v in ids if not 0 <= v < K]
        if bad:
            raise ValueError(f"SceneIndex.{what}: class {bad[0]} outside 0..{K - 1}")
        if len(set(ids)) != len(ids):
            seen = set()
            dup = next(v for v in ids if v in seen or seen.add(v))
            raise ValueError(f"SceneIndex.{what}: class {dup} listed twice")
        return ids

    def _class_thresholds(self, threshold, m, what):
        """a float, [m] values or a tensor -> fp32 [m] on the device, without a host synchronisation: host values go
        through pinned memory and an asynchronous copy"""
        if isinstance(threshold, torch.Tensor) and threshold.is_cuda:
            thr = threshold.to(device=self.device, dtype=torch.float32).reshape(-1)
        elif isinstance(threshold, (int, float)) and not isinstance(threshold, bool):
            thr = torch.full((1,), float(threshold), dtype=torch.float32, device=self.device)
        else:
            host = torch.as_tensor(threshold, dtype=torch.float32).reshape(-1)
            thr = host.pin_memory().to(self.device, non_blocking=True)
        if thr.numel() == 1:
            thr = thr.expand(m)
        if thr.numel() != m:
            raise ValueError(f"SceneIndex.{what}: {thr.numel()} thresholds for {m} classes")
        return thr.contiguous()

    def _label_counts(self, ids, thr):
        """osb_label_counts: int64 [S, len(ids)]"""
        S, dev, m = self.n_scenes, self.device, len(ids)
        with torch.cuda.device(dev):
            cnt = torch.empty((S, m), dtype=torch.int64, device=dev)
            ws_bytes = C.lib().osb_label_counts_workspace_bytes(self.vocab.shape[0], m)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
            C.call('osb_label_counts', C.ptr(self.row_label), C.ptr(self.row_label_score), C.ptr(self.row_scene),
                   self.n_rows, S, self.vocab.shape[0], (C.I64 * m)(*ids), m, C.ptr(thr), C.ptr(cnt), C.ptr(ws),
                   ws_bytes, C.stream_ptr())
        return cnt

    def class_counts(self, classes=None, threshold=None):
        """Per scene, the rows labelled each class: int64 [S, m], m = len(classes) (default: all K classes in order).
        Without ``threshold`` every row counts under its label, NaN scores included (the segmentation ``evaluate.py``
        counts); with ``threshold`` (a float or [m] values) only rows whose label score is not NaN and at or above
        threshold[j].  Refused above 2^27 counts.  No host synchronisation."""
        K = self._labelled('class_counts')
        ids = list(range(K)) if classes is None else self._classes(classes, K, 'class_counts')
        m, S = len(ids), self.n_scenes
        if S * m > MAX_COUNTS:
            raise ValueError(f"SceneIndex.class_counts: {S} scenes x {m} classes exceed {MAX_COUNTS} counts")
        thr = None if threshold is None else self._class_thresholds(threshold, m, 'class_counts')
        if S == 0:
            return torch.zeros((0, m), dtype=torch.int64, device=self.device)
        return self._label_counts(ids, thr)

    def class_regions(self, classes, threshold=None, max_regions=8, reach=1, min_voxels=1, hits=False, max_hits=2 ** 26):
        """``regions`` over the labels: the hits of class slot j are the rows labelled classes[j] whose label score is
        not NaN and at or above threshold[j] (default -inf), grouped into connected regions as ``regions`` groups them
        and ranked by the search key of their best hit.  Returns a ``RegionResult`` whose query axis is the position in
        ``classes``; any number of classes, in slices of 96.  Two host synchronisations, as ``regions``: the total hit
        count (refused above ``max_hits`` before the hit list is allocated) and the status word."""
        K = self._labelled('class_regions')
        if self.coords is None:
            raise RuntimeError("SceneIndex.class_regions: the index was built without coordinates (coords=True)")
        if self.n_scenes == 0:
            raise RuntimeError("SceneIndex.class_regions: the index is empty")
        if not 1 <= max_regions <= MAX_REGIONS:
            raise ValueError(f"SceneIndex.class_regions: max_regions={max_regions} outside 1..{MAX_REGIONS}")
        if reach not in (1, 2):
            raise ValueError(f"SceneIndex.class_regions: reach={reach} outside 1..2")
        if min_voxels < 1:
            raise ValueError(f"SceneIndex.class_regions: min_voxels={min_voxels} below 1")
        ids = self._classes(classes, K, 'class_regions')
        m, S, dev, R = len(ids), self.n_scenes, self.device, int(max_regions)
        thr = self._class_thresholds(float('-inf') if threshold is None else threshold, m, 'class_regions')
        slices = [(i, ids[i:i + MAX_QUERIES], thr[i:i + MAX_QUERIES].contiguous()) for i in range(0, m, MAX_QUERIES)]
        counts = [self._label_counts(ci, ts) for _, ci, ts in slices]

        def emit(si, h, cnt, key, hsc, status):
            _, ci, ts = slices[si]
            ws_bytes = C.lib().osb_label_hits_workspace_bytes(K, self.n_rows, S, len(ci))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
            C.call('osb_label_hits', C.ptr(self.row_label), C.ptr(self.row_label_score), C.ptr(self.row_scene),
                   self.n_rows, S, K, (C.I64 * len(ci))(*ci), len(ci), C.ptr(ts), C.ptr(cnt), h, C.ptr(key), C.ptr(hsc),
                   C.ptr(status), C.ptr(ws), ws_bytes, C.stream_ptr())

        return self._grow('class_regions', 'the label counts', [(q0, len(ci)) for q0, ci, _ in slices], counts, emit,
                          R, reach, min_voxels, hits, max_hits)

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

        def emit(si, h, cnt, key, hsc, status):
            _, qs, ts = slices[si]
            if qs.data_ptr() % 16:
                qs = qs.clone()
            ws_bytes = C.lib().osb_search_hits_workspace_bytes(S, qs.shape[0], h)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
            sfx, operand = self._operand()
            C.call('osb_search_hits' + sfx, *operand, C.ptr(self.row_scene), self.n_rows, self.channels,
                   (C.I64 * (S + 1))(*self._off), S, C.ptr(qs), qs.shape[0], C.ptr(ts), C.ptr(cnt), h, C.ptr(key),
                   C.ptr(hsc), C.ptr(status), C.ptr(ws), ws_bytes, C.stream_ptr())

        return self._grow('regions', "the search's counts", [(q0, qs.shape[0]) for q0, qs, _ in slices], counts, emit,
                          R, reach, min_voxels, hits, max_hits)

    def _grow(self, what, counted_by, slices, counts, emit, R, reach, min_voxels, hits, max_hits):
        """The tail of ``regions`` and ``class_regions``: per slice (q0, m) with counts [S, m], read the hit totals (host
        sync 1), refuse above max_hits, allocate the hit list, fill it with emit(slice, n_hits, counts, key, score,
        status), grow the regions with ``osb_regions``, and read the status word (host sync 2)."""
        S, dev = self.n_scenes, self.device
        with torch.cuda.device(dev):
            totals = [int(t) for t in torch.stack([c.sum() for c in counts]).tolist()]      # host sync 1
        total = sum(totals)
        if total > max_hits:
            raise RuntimeError(f"SceneIndex.{what}: {total} hits exceed max_hits={max_hits}; raise the threshold or "
                               f"max_hits")
        parts = []
        with torch.cuda.device(dev):
            status = torch.zeros(1, dtype=torch.int32, device=dev)
            for si, ((q0, m), cnt, h) in enumerate(zip(slices, counts, totals)):
                key = torch.empty(h, dtype=torch.int64, device=dev)
                hsc = torch.empty(h, dtype=torch.float16, device=dev)
                if h:
                    emit(si, h, cnt, key, hsc, status)
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
            raise RuntimeError(f"SceneIndex.{what}: a hit's coordinate lies outside |x|, |y|, |z| < 2^17 - 256")
        if st & C_ST_DUP:
            raise RuntimeError(f"SceneIndex.{what}: two hits of one (scene, query) share a voxel (duplicate coordinates)")
        if st:
            raise RuntimeError(f"SceneIndex.{what}: the hit list does not match {counted_by} (status {st})")
        if len(parts) == 1:
            return RegionResult(*parts[0])
        cat = lambda j, d: None if parts[0][j] is None else torch.cat([p[j] for p in parts], dim=d)   # noqa: E731
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


MAX_WORLD = 64        # OSB_SHARD_MAX_WORLD
MAX_SHARD_QUERIES = 65535    # OSB_SHARD_MAX_QUERIES

Directory = namedtuple('Directory', 'owner local rows base n_local names')
Directory.__doc__ = """Per global scene id: owner rank, local scene on that rank, row count, first global row (lists of
length S); n_local: scenes per rank; names: per global id."""


def build_directory(ids, rows, names, channels, storage, group=None):
    """The directory of a sharded index, built collectively: one ``all_gather_object`` of every rank's (global ids, row
    counts, names, width, storage), checked alike on every rank, so that a refusal is the same ValueError everywhere.
    The ids over the group must be exactly 0 .. S-1, the widths and storages equal.  No device work: this runs over any
    backend and without a GPU."""
    import torch.distributed as dist
    world = dist.get_world_size(group)
    mine = ([int(i) for i in ids], [int(r) for r in rows], list(names), int(channels), str(storage))
    every = [None] * world
    dist.all_gather_object(every, mine, group=group)
    for what, j in (('widths', 3), ('storages', 4)):
        vals = [e[j] for e in every]
        if len(set(vals)) > 1:
            raise ValueError(f"ShardedSceneIndex: the {what} differ over the group (per rank: {vals})")
    S = sum(len(e[0]) for e in every)
    owner, local, count = [None] * S, [None] * S, [None] * S
    out_of_range = []
    for w, (ids_w, rows_w, _, _, _) in enumerate(every):
        for j, (g, n) in enumerate(zip(ids_w, rows_w)):
            if not 0 <= g < S:
                out_of_range.append(g)
                continue
            if owner[g] is not None:
                raise ValueError(f"ShardedSceneIndex: scene id {g} is held twice (ranks {owner[g]} and {w})")
            owner[g], local[g], count[g] = w, j, n
    if out_of_range:
        missing = [g for g in range(S) if owner[g] is None]
        raise ValueError(f"ShardedSceneIndex: the scene ids over the group must be 0 .. {S - 1}; id {missing[0]} is "
                         f"missing (ids outside the range: {sorted(out_of_range)[:8]})")
    base, run = [], 0
    for n in count:
        base.append(run)
        run += n
    if run >= 2 ** 48:
        raise ValueError(f"ShardedSceneIndex: {run} rows over the group; the merge keys hold global rows below 2^48")
    gnames = [every[owner[g]][2][local[g]] for g in range(S)]
    return Directory(owner, local, count, base, [len(e[0]) for e in every], gnames)


def _rotate(t, a, o, e):
    """Move rows t[o:e] to t[a:a + e - o] and rows t[a:o] up behind them, on the device: the tail is copied aside, and
    the rows in between move in chunks from the top down through a bounce buffer (copies of overlapping memory are not
    allowed), at most 2^16 rows at a time."""
    n = e - o
    if o == a:
        return
    tail = t[o:e].clone()
    step = max(n, 1 << 16)
    buf = None if step == n else torch.empty((min(step, o - a),) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    hi = o
    while hi > a:
        lo = max(a, hi - step)
        if buf is None:
            t[lo + n:hi + n].copy_(t[lo:hi])              # n rows apart, at most n rows long: no overlap
        else:
            b = buf[:hi - lo]
            b.copy_(t[lo:hi])
            t[lo + n:hi + n].copy_(b)
        hi = lo
    t[a:a + n].copy_(tail)


class ShardedSceneIndex:
    """One database of scenes spread over the ranks of a process group (``process_group=None``: the default group).

    Each rank owns a ``SceneIndex`` (``local``) of the given capacity, width, storage and coordinates, and holds the
    scenes it added.  ``add`` is local and takes the scene's global id.  ``query``, ``regions`` and ``sync`` are
    collectives: every rank calls them in the same order with the same arguments.  Their outputs are, on every rank,
    bit for bit those of one ``SceneIndex`` that adds every scene in ascending global id, whatever the assignment of
    scenes to ranks and the order of the local adds.

    The directory (global id -> owner rank, local scene, row count, first global row) is built by ``sync``: one
    ``all_gather_object`` and one host synchronisation per change of the index.  ``query`` and ``regions`` call it on a
    rank that has added since the last build (or never built it), which covers the usual case of every rank adding its
    share before the first query.  A rank cannot learn of another rank's add without a host round trip, which ``query``
    does not make: after adds on some ranks only, call ``sync()`` on every rank.

    A rank keeps its scenes in ascending global id, so that its local row order is the global row order: ties inside
    a rank's top-k then fall as they fall in the single index.  An ``add`` out of that order moves the rows of the
    rank's scenes with higher ids up on the device (cost proportional to them; ``DistributedSampler`` with
    ``shuffle=False`` never does it)."""

    def __init__(self, capacity_rows, channels=768, process_group=None, device=None, coords=False, storage='fp16'):
        import torch.distributed as dist
        if not dist.is_available() or not dist.is_initialized():
            raise RuntimeError("ShardedSceneIndex: torch.distributed is not initialised")
        self.group = process_group if process_group is not None else dist.group.WORLD
        self.rank, self.world = dist.get_rank(self.group), dist.get_world_size(self.group)
        if self.world > MAX_WORLD:
            raise ValueError(f"ShardedSceneIndex: {self.world} ranks; at most {MAX_WORLD}")
        self.local = SceneIndex(capacity_rows, channels, device=device, coords=coords, storage=storage)
        self.device = self.local.device
        self._ids = []              # global id of each local scene, ascending (= the local scene order)
        self._dir = None

    # ------------------------------------------------------------------ local
    def add(self, rows, scene_id, name=None, coords=None):
        """Add one scene with its global id ``scene_id`` to this rank's shard; rows and coordinates are validated as in
        ``SceneIndex.add``.  Local: no collective, no host synchronisation.  Returns ``scene_id``."""
        if isinstance(scene_id, bool):
            raise TypeError("ShardedSceneIndex.add: scene_id must be an integer")
        try:
            sid = operator.index(scene_id)
        except TypeError:
            raise TypeError(f"ShardedSceneIndex.add: scene_id must be an integer (got {type(scene_id).__name__})")
        L = self.local
        p = bisect.bisect_right(self._ids, sid)
        s = L.add(rows, name=name, coords=coords)
        if p < s:
            self._move_last_scene(p)
        self._ids.insert(p, sid)
        self._dir = None
        return sid

    def _move_last_scene(self, p):
        """the local index's last scene becomes local scene p; the scenes p .. move up by one"""
        L = self.local
        off, S = L._off, L.n_scenes
        a, o, e = off[p], off[-2], off[-1]
        n = e - o
        for t in (L.rows, L.codes, L.row_exp, L.coords, L.row_scene):
            if t is not None:
                _rotate(t, a, o, e)
        L.row_scene[a + n:e] += 1
        L.row_scene[a:a + n].fill_(p)
        L._off_dev[p + 1:S + 1] = L._off_dev[p:S] + n
        L._off[:] = off[:p + 1] + [x + n for x in off[p:S]]
        L.names.insert(p, L.names.pop())

    # ------------------------------------------------------------------ directory
    def sync(self):
        """Build the directory (collective; one host synchronisation).  Raises the same ValueError on every rank when
        the ids over the group are not exactly 0 .. S-1, or the widths or storages differ."""
        L = self.local
        rows = [b - a for a, b in zip(L._off[:-1], L._off[1:])]
        with torch.cuda.device(self.device):
            d = build_directory(self._ids, rows, L.names, L.channels, L.storage, self.group)
            S, smax = len(d.owner), max(d.n_local)
            dev = self.device
            self._gid = torch.tensor(self._ids, dtype=torch.int64, device=dev)
            self._base = torch.tensor(d.base if S else [0], dtype=torch.int64, device=dev)
            self._place = torch.tensor([d.owner[g] * smax + d.local[g] for g in range(S)], dtype=torch.int64, device=dev)
        self._smax = smax
        self._dir = d

    def _directory(self):
        if self._dir is None:
            raise RuntimeError("ShardedSceneIndex: the directory is out of date; call sync() on every rank")
        return self._dir

    @property
    def n_scenes(self):
        """scenes over the group, as of the last directory build"""
        return len(self._directory().owner)

    @property
    def names(self):
        """names by global id, as of the last directory build"""
        return list(self._directory().names)

    def owner(self, scene_id):
        """the rank holding global scene ``scene_id``"""
        d = self._directory()
        if not 0 <= scene_id < len(d.owner):
            raise IndexError(f"ShardedSceneIndex.owner: scene id {scene_id} outside 0 .. {len(d.owner) - 1}")
        return d.owner[scene_id]

    def _ready(self, what):
        if self._dir is None:
            self.sync()
        if not self._dir.owner:
            raise RuntimeError(f"ShardedSceneIndex.{what}: the index is empty")

    # ------------------------------------------------------------------ merge helpers
    def _gather(self, x):
        """[world, *x.shape]: x of every rank"""
        import torch.distributed as dist
        out = [torch.empty_like(x) for _ in range(self.world)]
        dist.all_gather(out, x.contiguous(), group=self.group)
        return torch.stack(out)

    def _keys(self, score, scene, row):
        """global merge keys and global scene ids of decoded local results (osb_shard_keys)"""
        d = self._dir
        key, gsc = torch.empty_like(scene), torch.empty_like(scene)
        C.call('osb_shard_keys', C.ptr(score.contiguous()), C.ptr(scene.contiguous()), C.ptr(row.contiguous()),
               scene.numel(), C.ptr(self._gid) if self._gid.numel() else None, self._gid.numel(), C.ptr(self._base),
               len(d.owner), sum(d.rows), C.ptr(key), C.ptr(gsc), C.stream_ptr())
        return key, gsc

    def _merge(self, keys):
        """keys int64 [world, nq, m] -> winners int64 [nq, m], positions w * m + j (osb_shard_merge)"""
        W, nq, m = keys.shape
        win = torch.empty((nq, m), dtype=torch.int64, device=self.device)
        C.call('osb_shard_merge', C.ptr(keys.contiguous()), W, nq, m, C.ptr(win), C.stream_ptr())
        return win

    @staticmethod
    def _take(cols, win):
        """cols [ncol, world, nq, m], winners [nq, m] -> [ncol, nq, m]"""
        ncol, W, nq, m = cols.shape
        flat = cols.permute(0, 2, 1, 3).reshape(ncol, nq, W * m)
        return flat.gather(2, win.unsqueeze(0).expand(ncol, nq, m))

    def _per_scene(self, cols):
        """cols [ncol, world, smax, nq] -> [ncol, S, nq] in global id order"""
        ncol, W, smax, nq = cols.shape
        return cols.reshape(ncol, W * smax, nq).index_select(1, self._place)

    def _pad_scenes(self, ts, nq):
        """local per-scene tensors [S_r, nq] (int64) -> [ncol, smax, nq]"""
        out = torch.zeros((len(ts), self._smax, nq), dtype=torch.int64, device=self.device)
        for i, t in enumerate(ts):
            out[i, :t.shape[0]] = t
        return out

    @staticmethod
    def _bits(h):
        return h.view(torch.int16).long()

    @staticmethod
    def _half(x):
        return x.to(torch.int16).view(torch.float16)

    # ------------------------------------------------------------------ collectives
    def query(self, queries, k=1, threshold=None):
        """``SceneIndex.query`` over the whole group (collective): a ``SearchResult`` whose ``scene`` is the global id and
        whose per-scene outputs are [S, nq] by global id, equal bit for bit to the single index's.  With NCCL no host
        synchronisation once the directory is built."""
        if not 1 <= k <= MAX_K:
            raise ValueError(f"ShardedSceneIndex.query: k={k} outside 1..{MAX_K}")
        L = self.local
        q = L._queries(queries, 'query')
        nq = q.shape[0]
        if nq > MAX_SHARD_QUERIES:
            raise ValueError(f"ShardedSceneIndex.query: nq={nq} above {MAX_SHARD_QUERIES}; query in slices")
        thr = None if threshold is None else L._thresholds(threshold, nq, 'query')
        self._ready('query')
        dev = self.device
        with torch.cuda.device(dev):
            if L.n_scenes:
                res = L.query(q, k=k, threshold=thr)
            else:
                res = SearchResult(torch.full((nq, k), float('-inf'), dtype=torch.float16, device=dev),
                                   torch.full((nq, k), -1, dtype=torch.int64, device=dev),
                                   torch.full((nq, k), -1, dtype=torch.int64, device=dev),
                                   torch.empty((0, nq), dtype=torch.float16, device=dev),
                                   torch.empty((0, nq), dtype=torch.int64, device=dev),
                                   None if thr is None else torch.empty((0, nq), dtype=torch.int64, device=dev))
            key, gsc = self._keys(res.score, res.scene, res.row)
            top = torch.stack([key, gsc, res.row, self._bits(res.score)])                      # [4, nq, k]
            per = [self._bits(res.scene_max), res.scene_argmax] + ([] if thr is None else [res.scene_count])
            per = self._pad_scenes(per, nq)                                                      # [ncol, smax, nq]
            g = self._gather(torch.cat([top.reshape(-1), per.reshape(-1)]))
            W = self.world
            top_g = g[:, :top.numel()].reshape(W, 4, nq, k).transpose(0, 1)
            win = self._merge(top_g[0])
            dec = self._take(top_g[1:], win)
            sc = self._per_scene(g[:, top.numel():].reshape(W, per.shape[0], self._smax, nq).transpose(0, 1))
            return SearchResult(self._half(dec[2]), dec[0], dec[1], self._half(sc[0]), sc[1],
                                None if thr is None else sc[2])

    def regions(self, queries, threshold, max_regions=8, reach=1, min_voxels=1, hits=False, max_hits=2 ** 26):
        """``SceneIndex.regions`` over the whole group (collective), equal bit for bit to the single index's: ranked
        regions by global id, ``n_regions`` [S, nq], and with ``hits=True`` the hit list sorted by (query, global row),
        ``hit_region`` the rank in the merged list.  Two host synchronisations, as the single index: one read of every
        rank's hit totals (which size the hit gather; refused above ``max_hits`` summed over the group) and one read of
        the status word OR-ed over the group.  Both refusals are raised on every rank."""
        L = self.local
        if L.coords is None:
            raise RuntimeError("ShardedSceneIndex.regions: the index was built without coordinates (coords=True)")
        if not 1 <= max_regions <= MAX_REGIONS:
            raise ValueError(f"ShardedSceneIndex.regions: max_regions={max_regions} outside 1..{MAX_REGIONS}")
        if reach not in (1, 2):
            raise ValueError(f"ShardedSceneIndex.regions: reach={reach} outside 1..2")
        if min_voxels < 1:
            raise ValueError(f"ShardedSceneIndex.regions: min_voxels={min_voxels} below 1")
        q = L._queries(queries, 'regions')
        nq, dev, R, W = q.shape[0], self.device, int(max_regions), self.world
        thr = L._thresholds(threshold, nq, 'regions')
        self._ready('regions')
        S, Sr, smax = self.n_scenes, L.n_scenes, self._smax
        slices = [(i, q[i:i + MAX_QUERIES].contiguous(), thr[i:i + MAX_QUERIES].contiguous())
                  for i in range(0, nq, MAX_QUERIES)]
        with torch.cuda.device(dev):
            counts = [L._query(qs, 1, ts).scene_count for _, qs, ts in slices] if Sr else None
            mine = torch.stack([c.sum() for c in counts]) if Sr else torch.zeros(len(slices), dtype=torch.int64, device=dev)
            totals = self._gather(mine).tolist()                                          # host sync 1
        total = sum(map(sum, totals))
        if total > max_hits:
            raise RuntimeError(f"ShardedSceneIndex.regions: {total} hits over the group exceed max_hits={max_hits}; raise "
                               f"the threshold or max_hits")
        parts = []
        with torch.cuda.device(dev):
            status = torch.zeros(1, dtype=torch.int32, device=dev)
            for si, (q0, qs, ts) in enumerate(slices):
                m = qs.shape[0]
                h = totals[self.rank][si]
                out, hit_out, hsc = self._local_regions(qs, ts, counts[si] if Sr else None, h, R, reach, min_voxels,
                                                        hits, status)
                key, gsc = self._keys(out[0], out[1], out[2])
                reg = torch.cat([torch.stack([key, gsc, out[2], out[3], self._bits(out[0])]),
                                 out[4].long().permute(2, 0, 1), out[5].long().permute(2, 0, 1)])   # [11, m, R]
                per = self._pad_scenes([out[6]], m)
                flat = [reg.reshape(-1), per.reshape(-1)]
                hmax = max(t[si] for t in totals)
                if hits and hmax:
                    hl = torch.zeros((7, hmax), dtype=torch.int64, device=dev)
                    if h:
                        hg = self._gid[hit_out[1]]
                        hl[:, :h] = torch.stack([hit_out[0], self._base[hg] + hit_out[2], torch.full_like(hg, self.rank),
                                                 hit_out[3], hg, hit_out[2], self._bits(hsc)])
                    flat.append(hl.reshape(-1))
                g = self._gather(torch.cat(flat))
                n_reg, n_per = reg.numel(), per.numel()
                reg_g = g[:, :n_reg].reshape(W, 11, m, R).transpose(0, 1)
                win = self._merge(reg_g[0])
                dec = self._take(reg_g[1:], win)
                box = dec[4:].permute(1, 2, 0).to(torch.int32)                              # [m, R, 6]
                n_regions = self._per_scene(g[:, n_reg:n_reg + n_per].reshape(W, 1, smax, m).transpose(0, 1))[0]
                res = [self._half(dec[3]), dec[0], dec[1], dec[2], box[..., :3].contiguous(), box[..., 3:].contiguous(),
                       n_regions]
                if hits:
                    H = sum(t[si] for t in totals)
                    if H:
                        hg_all = g[:, n_reg + n_per:].reshape(W, 7, hmax)
                        hl = torch.cat([hg_all[w, :, :t[si]] for w, t in enumerate(totals) if t[si]], dim=1)
                        order = torch.empty(H, dtype=torch.int64, device=dev)
                        region = torch.empty(H, dtype=torch.int64, device=dev)
                        ws_bytes = C.lib().osb_shard_hits_workspace_bytes(H)
                        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
                        C.call('osb_shard_hits', C.ptr(hl[0].contiguous()), C.ptr(hl[1].contiguous()),
                               C.ptr(hl[2].contiguous()), C.ptr(hl[3].contiguous()), H, W, m, R, C.ptr(win),
                               C.ptr(order), C.ptr(region), C.ptr(ws), ws_bytes, C.stream_ptr())
                        del ws
                        hs = hl.index_select(1, order)
                        res += [hs[0] + q0, hs[4], hs[5], self._half(hs[6]), region]
                    else:
                        res += [torch.empty(0, dtype=torch.int64, device=dev)] * 3 + \
                               [torch.empty(0, dtype=torch.float16, device=dev),
                                torch.empty(0, dtype=torch.int64, device=dev)]
                else:
                    res += [None] * 5
                parts.append(res)
            st = 0
            for v in self._gather(status).reshape(-1).tolist():                          # host sync 2
                st |= int(v)
        if st & C_ST_RANGE:
            raise RuntimeError("ShardedSceneIndex.regions: a hit's coordinate lies outside |x|, |y|, |z| < 2^17 - 256")
        if st & C_ST_DUP:
            raise RuntimeError("ShardedSceneIndex.regions: two hits of one (scene, query) share a voxel (duplicate "
                               "coordinates)")
        if st:
            raise RuntimeError(f"ShardedSceneIndex.regions: the hit list does not match the search's counts (status {st})")
        if len(parts) == 1:
            return RegionResult(*parts[0])
        cat = lambda j, d: None if parts[0][j] is None else torch.cat([p[j] for p in parts], dim=d)   # noqa: E731
        return RegionResult(*[cat(j, 1 if j == 6 else 0) for j in range(12)])

    def _local_regions(self, qs, ts, cnt, h, R, reach, min_voxels, hits, status):
        """this rank's regions of one query slice, the steps of SceneIndex.regions: (region outputs with local scene
        ids, local hit list (query, local scene, row, local region rank) or None, hit scores)"""
        L, dev, m = self.local, self.device, qs.shape[0]
        if not L.n_scenes:
            out = [torch.full((m, R), float('-inf'), dtype=torch.float16, device=dev)] + \
                  [torch.full((m, R), -1, dtype=torch.int64, device=dev) for _ in range(2)] + \
                  [torch.zeros((m, R), dtype=torch.int64, device=dev)] + \
                  [torch.zeros((m, R, 3), dtype=torch.int32, device=dev) for _ in range(2)] + \
                  [torch.empty((0, m), dtype=torch.int64, device=dev)]
            return out, None, None
        S = L.n_scenes
        if qs.data_ptr() % 16:
            qs = qs.clone()
        key = torch.empty(h, dtype=torch.int64, device=dev)
        hsc = torch.empty(h, dtype=torch.float16, device=dev)
        if h:
            ws_bytes = C.lib().osb_search_hits_workspace_bytes(S, m, h)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
            sfx, operand = L._operand()
            C.call('osb_search_hits' + sfx, *operand, C.ptr(L.row_scene), L.n_rows, L.channels,
                   (C.I64 * (S + 1))(*L._off), S, C.ptr(qs), m, C.ptr(ts), C.ptr(cnt), h, C.ptr(key), C.ptr(hsc),
                   C.ptr(status), C.ptr(ws), ws_bytes, C.stream_ptr())
            del ws
        out = [torch.empty((m, R), dtype=torch.float16, device=dev)] + \
              [torch.empty((m, R), dtype=torch.int64, device=dev) for _ in range(3)] + \
              [torch.empty((m, R, 3), dtype=torch.int32, device=dev) for _ in range(2)] + \
              [torch.empty((S, m), dtype=torch.int64, device=dev)]
        hit_out = [torch.empty(h, dtype=torch.int64, device=dev) for _ in range(4)] if hits else [None] * 4
        ws_bytes = C.lib().osb_regions_workspace_bytes(h)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev) if h else None
        C.call('osb_regions', C.ptr(key), C.ptr(hsc), h, C.ptr(L.coords), C.ptr(L.row_scene), C.ptr(L._off_dev),
               L.n_rows, S, m, R, int(reach), int(min_voxels), *[C.ptr(t) for t in out], *[C.ptr(t) for t in hit_out],
               C.ptr(status), C.ptr(ws), ws_bytes, C.stream_ptr())
        return out, hit_out, hsc


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
