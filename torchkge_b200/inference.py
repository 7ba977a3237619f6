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

Extension: ``shard=EntityShard | QueryShard`` spreads the work over the ranks of a process group
(host logic in ``engine.topk_entity_inference`` / ``topk_relation_inference``, DESIGN.md section 6);
every rank ends with the full results, equal to those of one unsharded call.

Deviation, on purpose: the reference stores the scores with ``self.scores[i * b_size, (i + 1) *
b_size] = ...`` (inference.py:151, 246) -- an index pair instead of a slice, which raises
IndexError for every usual argument.  Here ``scores[i]`` holds the scores of ``predictions[i]``.
"""
import torch

from . import _lib
from .engine import TOPK_CHUNK, default_engine, shard_spec, topk_entity_inference, topk_relation_inference
from .exceptions import WrongArgumentsError

#: queries per top-k call
_MAX_QUERIES_PER_CALL = TOPK_CHUNK


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


class EntityInference(object):
    """Infer the missing entity of (known entity, known relation) pairs.

    Parameters (torchkge/inference.py:183-201)
    ----------
    model: TransE / TransH / TransD / DistMult / RESCAL / ComplEx / RotatE model on a CUDA device.
    known_entities, known_relations: torch.LongTensor (n_facts,)
    top_k: int
    missing: 'tails' (complete (h, r, ?)) or 'heads' (complete (?, r, t))
    dictionary: optional mapping (known entity, relation) -> set of entities known to complete the
        pair (``kg.dict_of_tails`` for missing tails, ``kg.dict_of_heads`` for missing heads);
        those are excluded from the predictions.
    shard: ``torchkge_b200.engine.EntityShard`` or ``QueryShard``, optional, keyword only
        (extension).  EntityShard: every rank of the group scans only its range of entity rows
        (``local_storage=True``: the model holds only those rows) and the per-rank top-k lists are
        merged on the device.  QueryShard (over ``len(known_entities)`` queries): every rank answers
        its contiguous slice of the queries against the whole (replicated) table.  Either way every
        rank ends up with the full results, equal to those of one unsharded call.

    Attributes: ``predictions`` LongTensor (n_facts, top_k), ``scores`` FloatTensor (n_facts, top_k),
    both on CPU after ``evaluate``.
    """

    def __init__(self, model, known_entities, known_relations, top_k=1, missing='tails', dictionary=None, *,
                 shard=None):
        if missing not in ('heads', 'tails'):
            raise WrongArgumentsError("missing entity should either be 'heads' or 'tails'")
        self.model = model
        self.known_entities = known_entities
        self.known_relations = known_relations
        self.missing = missing
        self.top_k = top_k
        self.dictionary = dictionary
        self.shard = shard
        self.predictions = torch.empty(size=(len(known_entities), top_k)).long()
        self.scores = torch.empty(size=(len(known_entities), top_k))

    def evaluate(self, b_size, verbose=True):
        """``b_size`` / ``verbose``: accepted for signature compatibility (chunking is by memory)."""
        spec = shard_spec(self.model, self.shard, "EntityInference.evaluate")
        dev = spec.ent0.device
        ents = self.known_entities.long().to(dev)
        rels = self.known_relations.long().to(dev)
        side = _lib.SIDE_TAIL if self.missing == 'tails' else _lib.SIDE_HEAD
        mask = None
        if self.dictionary is not None:
            mask = _mask_csr(self.dictionary, self.known_entities, self.known_relations)
        pred, vals = topk_entity_inference(spec, ents, rels, side, self.top_k, mask, shard=self.shard,
                                           engine=default_engine(), chunk=_MAX_QUERIES_PER_CALL)
        self.predictions, self.scores = pred.cpu(), vals.cpu()


class RelationInference(object):
    """Infer the missing relation of (entity 1, entity 2) pairs (torchkge/inference.py:78-155).

    model: TransE (L1/L2), TransH, TransD, DistMult or ComplEx model on a CUDA device.  dictionary: optional
    mapping (entity 1, entity 2) -> set of known relations (``kg.dict_of_rels``), excluded from
    the predictions.  Attributes: ``predictions`` (n_facts, top_k) long, ``scores`` float.
    shard: ``EntityShard`` or ``QueryShard``, optional, keyword only (extension).  The candidates
    are the relations, which every rank holds: under either type every rank answers a contiguous
    slice of the queries and the results are all-gathered; under EntityShard the rows of the two
    entities are first exchanged between the ranks that hold them.  Every rank ends up with the
    full results.
    """

    def __init__(self, model, entities1, entities2, top_k=1, dictionary=None, *, shard=None):
        self.model = model
        self.entities1 = entities1
        self.entities2 = entities2
        self.topk = top_k
        self.dictionary = dictionary
        self.shard = shard
        self.predictions = torch.empty(size=(len(entities1), top_k)).long()
        self.scores = torch.empty(size=(len(entities2), top_k))

    def evaluate(self, b_size, verbose=True):
        spec = shard_spec(self.model, self.shard, "RelationInference.evaluate")
        dev = spec.ent0.device
        e1, e2 = self.entities1.long().to(dev), self.entities2.long().to(dev)
        mask = None
        if self.dictionary is not None:
            mask = _mask_csr(self.dictionary, self.entities1, self.entities2)
        pred, vals = topk_relation_inference(spec, e1, e2, self.topk, mask, shard=self.shard,
                                             engine=default_engine(), chunk=_MAX_QUERIES_PER_CALL)
        self.predictions, self.scores = pred.cpu(), vals.cpu()
