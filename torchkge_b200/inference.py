"""``EntityInference`` / ``RelationInference`` with the reference's constructors and result
attributes (torchkge/inference.py:78-250): the top-k candidates that complete (h, r, ?),
(?, r, t) or (h, ?, t), optionally with the known facts of a dictionary masked out.

The selection runs inside the scan (``kge_topk_side``, csrc/topk.cu): the dense scan's "collect"
epilogue writes out only the candidates whose exact, ATen-order score is not below the query's
current k-th best, one chunk of candidate rows at a time, and a merge kernel keeps a sorted list of
k (score, id) pairs per query -- no (rows x candidates) score matrix exists.  Known facts are masked
with -inf exactly as ``filter_scores(..., true_idx=None)`` does (utils/modeling.py:76-102); results
are sorted descending as the reference's ``sort(descending=True)[:, :k]`` (the ORDER among exactly
tied scores is unspecified there; here: ascending candidate id, except that +0.0 ranks above -0.0
-- the returned scores keep their sign bit).

Deviation, on purpose: the reference stores the scores with ``self.scores[i * b_size, (i + 1) *
b_size] = ...`` (inference.py:151, 246) -- an index pair instead of a slice, which raises
IndexError for every usual argument.  Here ``scores[i]`` holds the scores of ``predictions[i]``.
"""
import torch

from . import _lib
from .engine import ModelSpec, default_engine, relation_spec
from .exceptions import WrongArgumentsError

_MAX_QUERIES_PER_CALL = 16384


def _mask_csr(dictionary, key1, key2):
    """CSR of dictionary[(key1[i], key2[i])] for every row (whole sets: true_idx is None), the ids
    of a row in ascending order (the merge kernel looks them up by bisection)."""
    offs, ids = [0], []
    get = dictionary.get if hasattr(dictionary, "get") else None
    for a, b in zip(key1.tolist(), key2.tolist()):
        s = get((a, b)) if get else dictionary[a, b]
        if s:
            ids.extend(sorted(s))
        offs.append(len(ids))
    return torch.tensor(offs, dtype=torch.int64), torch.tensor(ids, dtype=torch.int64)


def _topk_chunks(n, n_cand, top_k, topk_chunk, mask_csr, device):
    """Runs topk_chunk(lo, hi, mask) -> (pred, vals) over chunks of queries."""
    if top_k > n_cand:
        raise WrongArgumentsError("top_k = %d exceeds the %d candidates" % (top_k, n_cand))
    pred = torch.empty((n, top_k), dtype=torch.int64, device=device)
    vals = torch.empty((n, top_k), dtype=torch.float32, device=device)
    for lo in range(0, n, _MAX_QUERIES_PER_CALL):
        hi = min(n, lo + _MAX_QUERIES_PER_CALL)
        mask = None
        if mask_csr is not None:
            offs, ids = mask_csr
            a, b = int(offs[lo]), int(offs[hi])
            mask = ((offs[lo:hi + 1] - a).to(device), ids[a:b].to(device))
        pred[lo:hi], vals[lo:hi] = topk_chunk(lo, hi, mask)
    return pred, vals


class EntityInference(object):
    """Infer the missing entity of (known entity, known relation) pairs.

    Parameters (torchkge/inference.py:183-201)
    ----------
    model: TransE / DistMult / RESCAL / ComplEx / RotatE model on a CUDA device.
    known_entities, known_relations: torch.LongTensor (n_facts,)
    top_k: int
    missing: 'tails' (complete (h, r, ?)) or 'heads' (complete (?, r, t))
    dictionary: optional mapping (known entity, relation) -> set of entities known to complete the
        pair (``kg.dict_of_tails`` for missing tails, ``kg.dict_of_heads`` for missing heads);
        those are excluded from the predictions.

    Attributes: ``predictions`` LongTensor (n_facts, top_k), ``scores`` FloatTensor (n_facts, top_k),
    both on CPU after ``evaluate``.
    """

    def __init__(self, model, known_entities, known_relations, top_k=1, missing='tails', dictionary=None):
        if missing not in ('heads', 'tails'):
            raise WrongArgumentsError("missing entity should either be 'heads' or 'tails'")
        self.model = model
        self.known_entities = known_entities
        self.known_relations = known_relations
        self.missing = missing
        self.top_k = top_k
        self.dictionary = dictionary
        self.predictions = torch.empty(size=(len(known_entities), top_k)).long()
        self.scores = torch.empty(size=(len(known_entities), top_k))

    def evaluate(self, b_size, verbose=True):
        """``b_size`` / ``verbose``: accepted for signature compatibility (chunking is by memory)."""
        spec = ModelSpec.from_model(self.model)
        if not spec.ent0.is_cuda:
            raise _lib.KgeLibraryError("EntityInference.evaluate needs the model on a CUDA device; "
                                       "this package has no CPU execution path")
        dev = spec.ent0.device
        engine = default_engine()
        packed = engine.pack(spec)
        ents = self.known_entities.long().to(dev)
        rels = self.known_relations.long().to(dev)
        side = _lib.SIDE_TAIL if self.missing == 'tails' else _lib.SIDE_HEAD

        def topk_chunk(lo, hi, mask):
            rows = engine.gather_rows(spec, ents[lo:hi])
            return engine.topk_side(spec, packed, side, rows, rows, rels[lo:hi].contiguous(), self.top_k, mask)

        mask = None
        if self.dictionary is not None:
            mask = _mask_csr(self.dictionary, self.known_entities, self.known_relations)
        pred, vals = _topk_chunks(ents.shape[0], spec.n_rows, self.top_k, topk_chunk, mask, dev)
        self.predictions, self.scores = pred.cpu(), vals.cpu()


class RelationInference(object):
    """Infer the missing relation of (entity 1, entity 2) pairs (torchkge/inference.py:78-155).

    model: TransE (L1/L2), DistMult or ComplEx model on a CUDA device.  dictionary: optional
    mapping (entity 1, entity 2) -> set of known relations (``kg.dict_of_rels``), excluded from
    the predictions.  Attributes: ``predictions`` (n_facts, top_k) long, ``scores`` float.
    """

    def __init__(self, model, entities1, entities2, top_k=1, dictionary=None):
        self.model = model
        self.entities1 = entities1
        self.entities2 = entities2
        self.topk = top_k
        self.dictionary = dictionary
        self.predictions = torch.empty(size=(len(entities1), top_k)).long()
        self.scores = torch.empty(size=(len(entities2), top_k))

    def evaluate(self, b_size, verbose=True):
        spec = ModelSpec.from_model(self.model)
        if not spec.ent0.is_cuda:
            raise _lib.KgeLibraryError("RelationInference.evaluate needs the model on a CUDA device; "
                                       "this package has no CPU execution path")
        dev = spec.ent0.device
        engine = default_engine()
        e1, e2 = self.entities1.long().to(dev), self.entities2.long().to(dev)
        if spec.code == _lib.RESCAL:
            # candidates are relation matrices: dense (n, n_rel) scores, then the same selection kernels
            def topk_chunk(lo, hi, mask):
                hrows = engine.gather_rows(spec, e1[lo:hi]).view(hi - lo, spec.dim)
                trows = engine.gather_rows(spec, e2[lo:hi]).view(hi - lo, spec.dim)
                return engine.topk_dense(engine.rescal_rel_scores(spec, hrows, trows), self.topk, mask)

            mask = None
            if self.dictionary is not None:
                mask = _mask_csr(self.dictionary, self.entities1, self.entities2)
            pred, vals = _topk_chunks(e1.shape[0], spec.n_rel, self.topk, topk_chunk, mask, dev)
            self.predictions, self.scores = pred.cpu(), vals.cpu()
            return
        rspec = relation_spec(spec)
        packed = engine.pack(rspec)

        def topk_chunk(lo, hi, mask):
            hrows, trows = engine.gather_rows(spec, e1[lo:hi]), engine.gather_rows(spec, e2[lo:hi])
            return engine.topk_side(rspec, packed, _lib.SIDE_REL, hrows, trows, None, self.topk, mask)

        mask = None
        if self.dictionary is not None:
            mask = _mask_csr(self.dictionary, self.entities1, self.entities2)
        pred, vals = _topk_chunks(e1.shape[0], rspec.n_rows, self.topk, topk_chunk, mask, dev)
        self.predictions, self.scores = pred.cpu(), vals.cpu()
