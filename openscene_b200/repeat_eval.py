"""Test-time repeat vote on the device: ``run/evaluate.py:385-425`` and ``run/eval_mink.py:167-216`` with
``test_repeats > 1``, without the per-repeat ``.cpu()`` of the score matrices.

The reference keeps, for every point of the dataset, the sum of its score rows over the repeats (``store = pred + store``)
and after each repeat takes ``store.float().max(1)[1]``.  Here every scene keeps that sum in a device store, allocated in
repeat 0 and updated in place: for the match products (evaluate.py) the add happens in the epilogue of the tensor-core
product (``osb_match_vote``), so a repeat's ``[N_pts, K]`` scores are never written to memory; for the fp32 logits of
eval_mink.py it is ``osb_vote_accumulate``.  The labels of the repeat and of the sum feed two device
``metric.ConfusionMeter`` s.  A repeat moves nothing to the host except the two confusion matrices in ``end_repeat``.

Bits: the fp16 store is one fp16 add rounded to nearest even per repeat, which is what the reference's CPU
``pred + store`` computes (a zero store turns -0 into +0; 60000 + 60000 is inf).  The fp32 store is one fp32 add per
repeat.  Labels follow torch's CPU ``max(1)[1]``: the first NaN of a row if it holds one, else the first maximum
(ties to the lowest index, -0 == +0).  NaN payloads are not part of the contract.

Memory: 2*K bytes per point for the fp16 store (K text classes; 40 B at K = 20) or 4*C bytes for the fp32 store
(C logits), plus 8 bytes for the accumulated label, for every point of the dataset, for as long as the vote lives.

nuScenes evaluates only the points with ``label != 255``.  Voting on all points and counting only the kept ones gives the
same labels on the kept points (each point's row is voted on its own), and the confusion matrix skips ground truth 255,
so the whole scene is passed as it is, with its full ground truth.

Usage (evaluate.py, ``feature_type='distill'``)::

    vote = RepeatVote(None, dataset=labelset_name, mapper=mapper)    # not len(labelset): it ends with 'unlabeled'
    for rep_i in range(args.test_repeats):
        vote.begin_repeat()
        for i, (coords, feat, label, feat_3d, mask, inds_reverse) in enumerate(val_data_loader):   # shuffle=False
            predictions = model(sinput)
            vote.match_distill(i, predictions, inds_reverse.cuda(), text_features, gt=label.cuda(),
                               nofeat=mask[inds_reverse].cuda() if mark_no_feature_to_unknown else None)
        current_iou, accumu_iou = vote.end_repeat(stdout=True)
"""
import torch

from . import _cabi as C
from . import matching, metric

MAX_K = 512            # columns of a voted row (osb_vote_accumulate)
MAX_K_MATCH = 480      # text rows of a match product (osb_match_scores / osb_match_vote: at most five 96-row passes)


class _Scene:
    __slots__ = ('n_pts', 'k', 'store', 'label_acc')

    def __init__(self, n_pts, k, store, label_acc):
        self.n_pts, self.k, self.store, self.label_acc = n_pts, k, store, label_acc


def _num_classes(dataset):
    for key, n in metric._DATASET_CLASSES:
        if key in dataset:
            return n
    raise NotImplementedError(f"RepeatVote: unknown dataset {dataset!r}")


class RepeatVote:
    """Device-resident vote over test-time repeats for one evaluation run.

    num_classes  metric classes (the confusion matrix size), or None
    dataset      the reference's dataset / labelset name: the class count is then the one ``metric.evaluate(...,
                 dataset=...)`` uses (20 for scannet_3d, 16 for nuscenes_3d, ...), and a ``num_classes`` that disagrees
                 with it is refused.  evaluate.py's ``labelset`` ends with the appended 'unlabeled', so ``len(labelset)``
                 is one more than the metric's classes: bind with ``RepeatVote(None, dataset=labelset_name)``.
    mapper       optional int tensor applied to both labels before counting (nuScenes detailed -> 16 classes)
    store_dtype  torch.float16 for the match products of evaluate.py, torch.float32 for eval_mink.py's logits

    Scenes are keyed by the loader's batch index ``i``; with ``shuffle=False`` it names the same scene in every repeat."""

    def __init__(self, num_classes, dataset=None, mapper=None, store_dtype=torch.float16, device='cuda'):
        if store_dtype not in (torch.float16, torch.float32):
            raise TypeError(f"RepeatVote: store_dtype must be torch.float16 or torch.float32, got {store_dtype}")
        if dataset is not None:
            n = _num_classes(dataset)
            if num_classes is not None and int(num_classes) != n:
                raise ValueError(f"RepeatVote: num_classes={num_classes} disagrees with dataset {dataset!r}, which the "
                                 f"metric evaluates over {n} classes (len(labelset) counts the appended 'unlabeled')")
            num_classes = n
        elif num_classes is None:
            raise ValueError("RepeatVote: give num_classes or dataset")
        self.num_classes = int(num_classes)
        self.dataset = dataset
        self.device = torch.device(device)
        self.mapper = None if mapper is None else torch.as_tensor(mapper).to(device=self.device, dtype=torch.int64)
        self.store_dtype = store_dtype
        self.scenes = {}
        self.repeat = -1
        self._open = False
        self._visited = set()
        self._n_gt = 0
        self.meter_cur = metric.ConfusionMeter(self.num_classes, self.device)
        self.meter_acc = metric.ConfusionMeter(self.num_classes, self.device)

    # ------------------------------------------------------------------ repeats
    def begin_repeat(self):
        if self._open:
            raise RuntimeError(f"RepeatVote.begin_repeat: repeat {self.repeat} has not ended; call end_repeat() first")
        for m in (self.meter_cur, self.meter_acc):
            m.full.zero_()
            m.bad.zero_()
        self.repeat += 1
        self._visited = set()
        self._n_gt = 0
        self._open = True

    def end_repeat(self, stdout=False):
        """(current_iou, accumulated_iou): the mean IoU of this repeat's labels and of the accumulated vote.  SYNC."""
        if not self._open:
            raise RuntimeError("RepeatVote.end_repeat: no repeat is open; call begin_repeat() first")
        missing = sorted(i for i in self.scenes if i not in self._visited)
        if missing:
            raise RuntimeError(f"RepeatVote.end_repeat: scene(s) {missing[:8]} of repeat 0 were not voted in repeat "
                               f"{self.repeat}; the reference's `pred + store` over the dataset would fail on the shape "
                               f"mismatch")
        cur = self.meter_cur.evaluate()
        acc = self.meter_acc.evaluate()
        self._open = False
        if stdout:
            metric.print_evaluation(self._n_gt, *acc)
        return cur[0], acc[0]

    def labels(self, i=None):
        """Accumulated (unmapped) labels, int64: of scene ``i``, or of all scenes in index order (eval_mink's pred.npy)."""
        if self.repeat < 0 or not self.scenes:
            raise RuntimeError("RepeatVote.labels: nothing has been voted yet")
        if i is not None:
            return self.scenes[i].label_acc.clone()
        return torch.cat([self.scenes[j].label_acc for j in sorted(self.scenes)])

    # ------------------------------------------------------------------ per scene
    def _slot(self, what, i, n_pts, k, dtype, gt, nofeat, max_k=MAX_K):
        """Every refusal happens here, before anything is launched.  A new scene's store is allocated here but the scene
        is registered only once its vote has been launched (``_count``)."""
        if not self._open:
            raise RuntimeError(f"RepeatVote.{what}: no repeat is open; call begin_repeat() first")
        if dtype != self.store_dtype:
            raise TypeError(f"RepeatVote.{what}: this vote keeps a {self.store_dtype} store and cannot add {dtype} "
                            f"rows (use one RepeatVote per store dtype)")
        if not 1 <= k <= max_k:
            raise ValueError(f"RepeatVote.{what}: K={k} outside 1..{max_k}")
        if self.mapper is not None and k > self.mapper.numel():
            raise ValueError(f"RepeatVote.{what}: K={k} labels but the mapper has {self.mapper.numel()} entries")
        if i in self._visited:
            raise RuntimeError(f"RepeatVote.{what}: scene {i} was already voted in repeat {self.repeat}; adding it "
                               f"twice would count it twice")
        sc = self.scenes.get(i)
        if sc is None and self.repeat > 0:
            raise RuntimeError(f"RepeatVote.{what}: scene {i} was not part of repeat 0; every repeat must visit the "
                               f"same scenes")
        if sc is not None and (sc.n_pts, sc.k) != (n_pts, k):
            raise ValueError(f"RepeatVote.{what}: scene {i} has {n_pts} points x K={k} in repeat {self.repeat} but "
                             f"{sc.n_pts} x K={sc.k} in repeat 0")
        if gt is not None and torch.as_tensor(gt).numel() != n_pts:
            raise ValueError(f"RepeatVote.{what}: gt has {torch.as_tensor(gt).numel()} labels for {n_pts} points")
        if nofeat is not None and torch.as_tensor(nofeat).numel() != n_pts:
            raise ValueError(f"RepeatVote.{what}: nofeat has {torch.as_tensor(nofeat).numel()} entries for {n_pts} points")
        if sc is None:
            sc = _Scene(n_pts, k, torch.zeros((n_pts, k), dtype=self.store_dtype, device=self.device),
                        torch.empty(n_pts, dtype=torch.int64, device=self.device))
        return sc

    def _count(self, i, label_cur, sc, gt, nofeat):
        """after the vote of scene ``i`` was launched: register the scene, count both labels"""
        self.scenes[i] = sc
        self._visited.add(i)
        if gt is None:
            return
        cur, acc = label_cur, sc.label_acc
        if self.mapper is not None:
            cur, acc = self.mapper[cur], self.mapper[acc]
        if nofeat is not None:
            missing = ~torch.as_tensor(nofeat).to(device=self.device, dtype=torch.bool).view(-1)
            cur = cur.masked_fill(missing, metric.NO_FEATURE_ID)
            acc = acc.masked_fill(missing, metric.NO_FEATURE_ID)
        self.meter_cur.update(cur, gt)
        self.meter_acc.update(acc, gt)
        self._n_gt += torch.as_tensor(gt).numel()

    def _inds(self, inds_reverse):
        if inds_reverse is None:
            return None
        return inds_reverse.to(device=self.device, dtype=torch.int64).contiguous()

    def _match(self, what, i, feat, inds_reverse, text, gt, nofeat):
        C.require_cuda(feat, 'features')
        feat = feat.contiguous()
        if feat.dtype not in (torch.float16, torch.float32):
            feat = feat.float()
        text = text.to(device=feat.device, dtype=torch.float16).contiguous()
        n_vox, c = feat.shape
        k = text.shape[0]
        if text.shape[1] != c:
            raise ValueError(f"RepeatVote.{what}: text embeddings have width {text.shape[1]}, features {c}")
        inv = self._inds(inds_reverse)
        n_pts = inv.shape[0] if inv is not None else n_vox
        sc = self._slot(what, i, n_pts, k, torch.float16, gt, nofeat, MAX_K_MATCH)
        label_cur = torch.empty(n_pts, dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            C.call('osb_match_vote', C.ptr(feat), int(feat.dtype == torch.float16), n_vox, c, C.ptr(inv), n_pts,
                   C.ptr(text), k, 0, None, C.ptr(sc.store), C.ptr(label_cur), C.ptr(sc.label_acc), C.stream_ptr())
        self._count(i, label_cur, sc, gt, nofeat)
        return label_cur

    def match_distill(self, i, predictions, inds_reverse, text, gt=None, nofeat=None):
        """evaluate.py:288-292 for scene ``i``: ``pred = predictions[inds_reverse].half() @ text.t()`` added into the vote.

        gt      per-point ground truth (counted in both confusion matrices), or None
        nofeat  the has-feature mask ``mask[inds_reverse]`` of ``mark_no_feature_to_unknown``: where it is False both
                labels count as 256 (evaluate.py:404-421)
        Returns this repeat's unmapped labels, int64 [N_pts]."""
        return self._match('match_distill', i, predictions, inds_reverse, text, gt, nofeat)

    def match_fusion(self, i, feat_3d, inds_reverse, text, gt=None, nofeat=None):
        """evaluate.py:293-296 (the fused 2-D features) for scene ``i``; as ``match_distill``."""
        return self._match('match_fusion', i, feat_3d, inds_reverse, text, gt, nofeat)

    def match_ensemble(self, i, predictions, feat_3d, inds_reverse, text, gt=None, nofeat=None):
        """evaluate.py:302-323 for scene ``i``: both cosine products pick each point's feature, and the final product
        is added into the vote.  Returns this repeat's unmapped labels."""
        C.require_cuda(predictions, 'features')
        predictions = predictions.contiguous().float()
        feat_3d = feat_3d.to(predictions.device)
        if feat_3d.dtype != torch.float16:
            feat_3d = feat_3d.half()
        feat_3d = feat_3d.contiguous()
        text = text.to(device=predictions.device, dtype=torch.float16).contiguous()
        n_vox, c = predictions.shape
        k = text.shape[0]
        if text.shape[1] != c or feat_3d.shape != predictions.shape:
            raise ValueError(f"RepeatVote.match_ensemble: shapes {tuple(predictions.shape)}, {tuple(feat_3d.shape)}, "
                             f"text {tuple(text.shape)} do not agree")
        inv = self._inds(inds_reverse)
        n_pts = inv.shape[0] if inv is not None else n_vox
        sc = self._slot('match_ensemble', i, n_pts, k, torch.float16, gt, nofeat, MAX_K_MATCH)
        _, _, smax2d = matching._scores(feat_3d, inv, text, normalize=True, want_scores=False, want_smax=True)
        _, _, smax3d = matching._scores(predictions, inv, text, normalize=True, want_scores=False, want_smax=True)
        label_cur = torch.empty(n_pts, dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            C.call('osb_match_ensemble_vote', C.ptr(predictions), C.ptr(feat_3d), n_vox, c, C.ptr(inv), n_pts,
                   C.ptr(smax3d), C.ptr(smax2d), C.ptr(text), k, None, C.ptr(sc.store), C.ptr(label_cur),
                   C.ptr(sc.label_acc), C.stream_ptr())
        self._count(i, label_cur, sc, gt, nofeat)
        return label_cur

    def add_logits(self, i, logits, inds_reverse, gt=None):
        """eval_mink.py:190-205 for scene ``i``: ``store += logits[inds_reverse]`` in the logits' precision (fp32 for
        MinkUNet's classifier head).  Returns this repeat's labels ``logits[inds_reverse].max(1)[1]``."""
        C.require_cuda(logits, 'logits')
        logits = logits.contiguous()
        if logits.dtype not in (torch.float16, torch.float32):
            logits = logits.float()
        n_src, k = logits.shape
        inv = self._inds(inds_reverse)
        n_pts = inv.shape[0] if inv is not None else n_src
        sc = self._slot('add_logits', i, n_pts, k, logits.dtype, gt, None)
        label_cur = torch.empty(n_pts, dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            C.call('osb_vote_accumulate', C.ptr(logits), int(logits.dtype == torch.float16), n_src, C.ptr(inv), n_pts,
                   k, C.ptr(sc.store), C.ptr(label_cur), C.ptr(sc.label_acc), C.stream_ptr())
        self._count(i, label_cur, sc, gt, None)
        return label_cur
