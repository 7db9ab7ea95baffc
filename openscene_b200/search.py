"""Search a database of scenes on the device (csrc/search.cu; DESIGN.md, "Scene search contract").

OpenScene's per-voxel features answer open-vocabulary queries over many scenes at once: rare-object search by name (CLIP
text rows) and image-based retrieval (CLIP image rows).  ``SceneIndex`` keeps the operand rows of many scenes in one
fixed device arena, and ``query`` scores every row against the queries on the tensor cores, with the bits
``osb_match_scores`` gives the same row, and returns

- the k best rows per query over the whole index (score, scene, row within the scene);
- per scene and query the best score and its row, and optionally how many rows score at or above a threshold.

The [N, nq] scores never exist in memory.  One memset and two launches serve up to 96 queries, and each such slice reads
the index once; more queries run slice after slice.  Nothing synchronises the host.
"""
from collections import namedtuple

import torch

from . import _cabi as C

MAX_QUERIES = 96      # OSB_SEARCH_MAX_QUERIES: one 96-column wgmma pass per launch
MAX_K = 32            # OSB_SEARCH_MAX_K

SearchResult = namedtuple('SearchResult', 'score scene row scene_max scene_argmax scene_count')
SearchResult.__doc__ = """score fp16 / scene int64 / row int64 [nq, k]: best first, (-inf, -1, -1) past the last non-NaN row;
scene_max fp16 / scene_argmax int64 [S, nq]: (-inf, -1) for a scene without a non-NaN score; scene_count int64 [S, nq]
(rows with float(score) >= threshold[q]) or None."""


class SceneIndex:
    """A fixed device arena of fp16 operand rows [capacity_rows, channels], filled scene after scene by ``add``.

    Scene ids follow the order of ``add``.  The arena never grows and is never re-copied."""

    def __init__(self, capacity_rows, channels=768, device=None):
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
        self.rows = torch.empty((self.capacity, self.channels), dtype=torch.float16, device=self.device)
        self.row_scene = torch.empty(self.capacity, dtype=torch.int32, device=self.device)
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
        """The rows [n, C] of one scene (a view into the arena)."""
        return self.rows[self._off[scene]:self._off[scene + 1]]

    def add(self, rows, name=None):
        """Append one scene's operand rows (fp16 [n, C]; fp32 is taken as ``.half()``, the 'distill' operand) and return
        its scene id.  An empty scene, a wrong width, dtype or device, or a full arena is refused before anything is
        copied."""
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
        o = self.n_rows
        if o + n > self.capacity:
            raise RuntimeError(f"SceneIndex.add: {n} rows do not fit ({self.capacity - o} of {self.capacity} left)")
        s = self.n_scenes
        self.rows[o:o + n].copy_(rows)                    # fp32 -> fp16 rounds to nearest even, as `.half()`
        self.row_scene[o:o + n].fill_(s)
        if s + 2 > self._off_dev.numel():
            grown = torch.zeros(2 * self._off_dev.numel(), dtype=torch.int64, device=self.device)
            grown[:self._off_dev.numel()].copy_(self._off_dev)
            self._off_dev = grown
        self._off_dev[s + 1] = o + n
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
            C.call('osb_search', C.ptr(self.rows), C.ptr(self.row_scene), self.n_rows, self.channels, off_host,
                   C.ptr(self._off_dev), S, C.ptr(q), nq, k, C.ptr(thr), C.ptr(score), C.ptr(scene), C.ptr(row),
                   C.ptr(smax), C.ptr(sarg), C.ptr(cnt), C.ptr(ws), ws_bytes, C.stream_ptr())
        return SearchResult(score, scene, row, smax, sarg, cnt)


def search_workspace_bytes(n_scenes, nq, k):
    """Device workspace of one launch pair (independent of the number of rows)."""
    return int(C.lib().osb_search_workspace_bytes(n_scenes, nq, k))
