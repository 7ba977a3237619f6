"""``LinkPredictionEvaluator`` with the reference's constructor, attributes and metric
methods (torchkge/evaluation.py:207-425).  ``evaluate`` hands the whole job -- scoring every
entity as head and as tail of every fact, discounting the filter sets, ranking -- to the
CUDA engine; no (batch, n_entities) score matrix exists at any point.
"""
from types import SimpleNamespace

import torch

from . import _lib
from .data import dict_filter_csr, filter_csr
from .engine import (DEFAULT_CHUNK, EntityShard, ModelSpec, ProjectedSpec, QueryShard, _by_query_slices,
                     _check_table, default_engine, rank_link_prediction, rank_link_prediction_projected,
                     rank_relation_prediction, refuse_projected_shard, relation_groups, score_triples_entity_sharded,
                     shard_spec)
from .exceptions import NotYetEvaluatedError


def _check_index_range(heads, tails, rels, n_ent, n_rel):
    """nn.Embedding raises on an out-of-range index; the kernels would read out of bounds.  The index
    tensors of a graph live on the host, so the check is a few microseconds there."""
    for name, x, hi in (("head", heads, n_ent), ("tail", tails, n_ent), ("relation", rels, n_rel)):
        if x.numel() and not x.is_cuda and (int(x.min()) < 0 or int(x.max()) >= hi):
            raise IndexError("%s index out of range [0, %d)" % (name, hi))


class LinkPredictionEvaluator(object):
    """Evaluate an embedding model by link prediction (Bordes et al. 2013).

    Parameters
    ----------
    model: a model of ``torchkge_b200.models`` (or the reference's class of the same name),
        living on a CUDA device.
    knowledge_graph: object exposing ``n_facts, head_idx, tail_idx, relations,
        dict_of_heads, dict_of_tails`` (``torchkge.data_structures.KnowledgeGraph`` or
        ``torchkge_b200.data.KnowledgeGraph``).
    shard: ``torchkge_b200.engine.EntityShard`` or ``QueryShard``, optional (extension).
        EntityShard: every rank of the group scans only its range of entity rows and the
        per-fact counters are summed with one all-reduce.  QueryShard: every rank ranks its
        contiguous slice of the facts against the whole (replicated) table and the rank vectors
        are all-gathered.  Either way all ranks end up with the full rank vectors.

    Attributes (as in the reference, evaluation.py:236-261)
    ----------
    rank_true_heads, rank_true_tails, filt_rank_true_heads, filt_rank_true_tails:
        torch.LongTensor (n_facts,), on CPU after ``evaluate``.
    evaluated: bool
    """

    def __init__(self, model, knowledge_graph, shard=None):
        self.model = model
        self.kg = knowledge_graph
        n = knowledge_graph.n_facts
        self.rank_true_heads = torch.empty(size=(n,)).long()
        self.rank_true_tails = torch.empty(size=(n,)).long()
        self.filt_rank_true_heads = torch.empty(size=(n,)).long()
        self.filt_rank_true_tails = torch.empty(size=(n,)).long()
        self.evaluated = False
        self.shard = shard
        self.last_stats = {}

    def evaluate(self, b_size, verbose=True):
        """Rank all facts of the graph.

        ``b_size`` is accepted for signature compatibility; as in the reference it never
        changes the result.  Here it does not bound memory either (nothing of size
        b_size x n_entities is allocated); facts are processed in chunks of
        ``engine.DEFAULT_CHUNK``.  ``verbose`` is accepted and ignored (no per-batch loop to
        report on).
        """
        if b_size is None or int(b_size) < 1:
            raise ValueError("b_size must be a positive integer")
        kg = self.kg
        spec = shard_spec(self.model, self.shard, "LinkPredictionEvaluator.evaluate", n=kg.n_facts)
        qshard = self.shard if isinstance(self.shard, QueryShard) else None
        eshard = None if qshard is not None else self.shard
        dev = spec.ent0.device
        heads, tails, rels = kg.head_idx, kg.tail_idx, kg.relations
        if qshard is not None:      # this rank's contiguous slice of the facts
            heads, tails, rels = qshard.slice(heads, tails, rels)
        n_here = int(heads.shape[0])
        _check_index_range(heads, tails, rels, spec.n_ent, spec.n_rel)
        h_d = heads.to(dev, non_blocking=True)
        t_d = tails.to(dev, non_blocking=True)
        r_d = rels.to(dev, non_blocking=True)
        stats = {"h2d_bytes": 8 * 3 * n_here, "d2h_bytes": 8 * (4 * kg.n_facts + 1)}
        projected = isinstance(spec, ProjectedSpec)
        if projected:
            # TransH and TransD rank the facts relation by relation: everything below, filter sets included, runs on
            # the facts sorted by relation; the ranks go back to fact order at the end
            order, order_host, groups = relation_groups(r_d, spec.n_rel)
            heads, tails, rels = heads[order_host], tails[order_host], rels[order_host]
            h_d, t_d, r_d = h_d[order], t_d[order], r_d[order]

        # Filter sets -> CSR (same per-row semantics as get_true_targets).  Built lazily: the
        # engine asks for them after the dense scans are enqueued, so host work overlaps the GPU.
        index = getattr(kg, "filter_index", None)
        if index is not None:
            # sorted-array filters (torchkge_b200.data.KnowledgeGraph): the index is resident on
            # the device (uploaded at first use, like weights); the per-row lists of this test set
            # come from searchsorted + gather on the device
            # ... once per (graph, test slice, device): the lists depend only on the graph, so they are
            # kept on the graph object like the index itself (keyed on the host index tensors)
            def from_index(which, k1, k2, true, k1_d, k2_d, true_d):
                def build():
                    cache = kg.__dict__.setdefault("_b200_filter_cache", {})
                    # identity of the host tensors + a cheap content fingerprint (in-place edits of a
                    # test set are unusual, but must not be served stale lists)
                    key = (which, str(dev), id(index), k1.data_ptr(), k2.data_ptr(), true.data_ptr(), n_here,
                           int(k1.sum()), int(k2.sum()), int(true.sum()))
                    hit = cache.get(key)
                    if hit is None:
                        while len(cache) >= 4:
                            cache.pop(next(iter(cache)))
                        hit = cache[key] = index.csr(which, k1_d, k2_d, true_d)
                    return hit
                return build
            csr_tail = from_index("tail", heads, rels, tails, h_d, r_d, t_d)
            csr_head = from_index("head", tails, rels, heads, t_d, r_d, h_d)
        else:
            # the reference's dictionaries (torchkge.data_structures.KnowledgeGraph): distinct
            # keys flattened once on the host, expanded on the device, cached on the graph
            def from_dicts(which, k1, k2, true):
                def build():
                    csr, nbytes = dict_filter_csr(kg, which, k1, k2, true, dev)
                    stats["h2d_bytes"] += nbytes
                    return csr
                return build
            csr_tail = from_dicts("tail", heads, rels, tails)
            csr_head = from_dicts("head", tails, rels, heads)
        engine = default_engine()
        if projected:
            lazy = rank_link_prediction_projected(spec, h_d, t_d, r_d, groups, csr_tail, csr_head, engine=engine,
                                                  chunk=DEFAULT_CHUNK, sync=False)
        else:
            lazy = rank_link_prediction(spec, h_d, t_d, r_d, csr_tail, csr_head, shard=eshard,
                                        engine=engine, chunk=DEFAULT_CHUNK, sync=False)

        def to_host(ranks, flag):
            flag = torch.zeros(1, dtype=torch.int64, device=dev) if flag is None else flag.long().view(1)
            if projected:      # back to fact order
                unsorted = [torch.empty_like(x) for x in ranks]
                for u, x in zip(unsorted, ranks):
                    u[order] = x
                ranks = unsorted
            if qshard is not None:
                ranks = qshard.all_gather(ranks)
                flag = qshard.all_reduce_sum(flag)   # every rank takes the same decision below
            return torch.cat([x.view(-1) for x in ranks] + [flag]).cpu()   # ONE device -> host copy

        host = to_host(lazy.ranks, lazy.overflow)
        if int(host[-1]) > 0:        # near-tie list overflow somewhere: exact recomputation
            host = to_host(lazy.get(flag_host=int(host[-1])), None)
        n = kg.n_facts
        self.last_stats = stats
        self.rank_true_heads, self.rank_true_tails = host[0:n], host[n:2 * n]
        self.filt_rank_true_heads, self.filt_rank_true_tails = host[2 * n:3 * n], host[3 * n:4 * n]
        self.evaluated = True

    def _check(self):
        if not self.evaluated:
            raise NotYetEvaluatedError('Evaluator not evaluated call '
                                       'LinkPredictionEvaluator.evaluate')

    def mean_rank(self):
        """(mean rank, filtered mean rank), heads and tails averaged (evaluation.py:310-330)."""
        self._check()
        raw = (self.rank_true_heads.float().mean() + self.rank_true_tails.float().mean()).item()
        filt = (self.filt_rank_true_heads.float().mean()
                + self.filt_rank_true_tails.float().mean()).item()
        return raw / 2, filt / 2

    def hit_at_k_heads(self, k=10):
        self._check()
        return ((self.rank_true_heads <= k).float().mean().item(),
                (self.filt_rank_true_heads <= k).float().mean().item())

    def hit_at_k_tails(self, k=10):
        self._check()
        return ((self.rank_true_tails <= k).float().mean().item(),
                (self.filt_rank_true_tails <= k).float().mean().item())

    def hit_at_k(self, k=10):
        """(Hits@k, filtered Hits@k), heads and tails averaged (evaluation.py:354-374)."""
        self._check()
        hh, fhh = self.hit_at_k_heads(k=k)
        th, fth = self.hit_at_k_tails(k=k)
        return (hh + th) / 2, (fhh + fth) / 2

    def mrr(self):
        """(MRR, filtered MRR), heads and tails averaged (evaluation.py:376-397)."""
        self._check()
        head = (self.rank_true_heads.float() ** (-1)).mean()
        tail = (self.rank_true_tails.float() ** (-1)).mean()
        fhead = (self.filt_rank_true_heads.float() ** (-1)).mean()
        ftail = (self.filt_rank_true_tails.float() ** (-1)).mean()
        return (head + tail).item() / 2, (fhead + ftail).item() / 2

    def print_results(self, k=None, n_digits=3):
        """Same report as the reference (evaluation.py:399-425)."""
        if k is None:
            k = 10
        if type(k) == int:
            k = [k]
        for i in k:
            print('Hit@{} : {} \t\t Filt. Hit@{} : {}'.format(
                i, round(self.hit_at_k(k=i)[0], n_digits),
                i, round(self.hit_at_k(k=i)[1], n_digits)))
        print('Mean Rank : {} \t Filt. Mean Rank : {}'.format(
            int(self.mean_rank()[0]), int(self.mean_rank()[1])))
        print('MRR : {} \t\t Filt. MRR : {}'.format(
            round(self.mrr()[0], n_digits), round(self.mrr()[1], n_digits)))


class RelationPredictionEvaluator(object):
    """Evaluate an embedding model by relation prediction (torchkge/evaluation.py:16-204): every
    fact's true relation is ranked against all relations, raw and filtered by
    ``knowledge_graph.dict_of_rels``.

    Parameters
    ----------
    model: TransE (L1/L2), TransH, TransD, DistMult, RESCAL, ComplEx or Analogy model on a CUDA device.
    knowledge_graph: object exposing ``n_facts, head_idx, tail_idx, relations, dict_of_rels``.
    directed: bool (default True).  False: both (h, ?, t) and (t, ?, h) are scored and ranked
        together against the directed true score (evaluation.py:99-107).
    shard: ``torchkge_b200.engine.EntityShard`` or ``QueryShard``, optional, keyword-only
        (extension).  The candidates are the relations, which every rank holds, so both forms split
        the facts over the ranks and all-gather the rank vectors.  QueryShard (over ``n_facts``):
        every rank ranks its contiguous slice of the facts, filtered by its slice of
        ``dict_of_rels``.  EntityShard with ``local_storage=True`` (the model holds only entity rows
        [lo, hi) and its row 0 is entity lo): per chunk of facts the h and t rows are exchanged by one
        all-reduce, then the chunk's facts are split as QueryShard splits them.  EntityShard with full
        storage: the facts are split as QueryShard splits them, no rows move.  Every rank ends with
        the rank vectors of the unsharded evaluator, exactly.

    Attributes: ``rank_true_rels``, ``filt_rank_true_rels`` (LongTensor (n_facts,), CPU after
    ``evaluate``), ``evaluated``, ``directed``.
    """

    def __init__(self, model, knowledge_graph, directed=True, *, shard=None):
        self.model = model
        self.kg = knowledge_graph
        self.directed = directed
        self.shard = shard
        self.rank_true_rels = torch.empty(size=(knowledge_graph.n_facts,)).long()
        self.filt_rank_true_rels = torch.empty(size=(knowledge_graph.n_facts,)).long()
        self.evaluated = False

    def evaluate(self, b_size, verbose=True):
        """``b_size`` / ``verbose`` are accepted for signature compatibility (see
        ``LinkPredictionEvaluator.evaluate``).  Under a shard, every rank of its group calls this."""
        if b_size is None or int(b_size) < 1:
            raise ValueError("b_size must be a positive integer")
        spec = shard_spec(self.model, self.shard, "RelationPredictionEvaluator.evaluate")
        dev = spec.ent0.device
        kg = self.kg
        _check_index_range(kg.head_idx, kg.tail_idx, kg.relations, spec.n_ent, spec.n_rel)
        h_d, t_d, r_d = (x.to(dev, non_blocking=True) for x in (kg.head_idx, kg.tail_idx, kg.relations))
        csr = filter_csr(kg.dict_of_rels, kg.head_idx, kg.tail_idx, kg.relations)
        csr = tuple(x.to(dev, non_blocking=True) for x in csr)
        rr, frr = rank_relation_prediction(spec, h_d, t_d, r_d, csr, directed=self.directed,
                                           engine=default_engine(), chunk=DEFAULT_CHUNK, shard=self.shard)
        self.rank_true_rels = rr.cpu()
        self.filt_rank_true_rels = frr.cpu()
        self.evaluated = True

    def _check(self):
        if not self.evaluated:
            raise NotYetEvaluatedError('Evaluator not evaluated call '
                                       'LinkPredictionEvaluator.evaluate')

    def mean_rank(self):
        """(mean rank, filtered mean rank) of the true relation (evaluation.py:114-131)."""
        self._check()
        return self.rank_true_rels.float().mean().item(), self.filt_rank_true_rels.float().mean().item()

    def hit_at_k(self, k=10):
        """(Hit@k, filtered Hit@k) (evaluation.py:133-154)."""
        self._check()
        return ((self.rank_true_rels <= k).float().mean().item(),
                (self.filt_rank_true_rels <= k).float().mean().item())

    def mrr(self):
        """(MRR, filtered MRR) (evaluation.py:156-174)."""
        self._check()
        return ((self.rank_true_rels.float() ** (-1)).mean().item(),
                (self.filt_rank_true_rels.float() ** (-1)).mean().item())

    def print_results(self, k=None, n_digits=3):
        """Same report as the reference (evaluation.py:176-204)."""
        if k is None:
            k = 10
        if k is not None and type(k) == int:
            print('Hit@{} : {} \t\t Filt. Hit@{} : {}'.format(
                k, round(self.hit_at_k(k=k)[0], n_digits), k, round(self.hit_at_k(k=k)[1], n_digits)))
        if k is not None and type(k) == list:
            for i in k:
                print('Hit@{} : {} \t\t Filt. Hit@{} : {}'.format(
                    i, round(self.hit_at_k(k=i)[0], n_digits), i, round(self.hit_at_k(k=i)[1], n_digits)))
        print('Mean Rank : {} \t Filt. Mean Rank : {}'.format(
            int(self.mean_rank()[0]), int(self.mean_rank()[1])))
        print('MRR : {} \t\t Filt. MRR : {}'.format(
            round(self.mrr()[0], n_digits), round(self.mrr()[1], n_digits)))


class TripletClassificationEvaluator(object):
    """Evaluate an embedding model by triplet classification (Socher et al. 2013),
    torchkge/evaluation.py:428-580: one threshold per relation (the best-scoring negative of the
    validation facts of that relation), then accuracy on the test facts and their negatives.

    Scores come from ``model.scoring_function`` (the CUDA per-triple scorer), negatives from
    ``PositionalNegativeSampler(kg_val, kg_test=kg_test)`` as in the reference; ``sampler`` may be
    replaced after construction.

    shard: ``torchkge_b200.engine.EntityShard`` or ``QueryShard``, optional, keyword-only
    (extension); every rank of its group makes the same calls.  EntityShard with
    ``local_storage=True`` (the model holds only entity rows [lo, hi)): per batch the h and t rows are
    exchanged by one all-reduce and every rank scores the batch with the same per-triple kernel.
    QueryShard, or EntityShard with full storage: every rank scores its contiguous slice of each score
    vector (split by that vector's length; the QueryShard's own ``n`` is not used) and the slices are
    all-gathered.  The negatives of every ``corrupt_kg`` call are rank 0's, sent to the other ranks in
    one collective, so that ranks seeded differently still agree.  ``get_scores`` returns the full
    score vector on every rank, equal bit for bit to the unsharded evaluator's; ``thresholds`` and
    ``accuracy`` are the same on every rank and equal those of an unsharded evaluator whose sampler
    draws what rank 0's sampler draws.
    """

    def __init__(self, model, kg_val, kg_test, *, shard=None):
        from .sampling import PositionalNegativeSampler
        refuse_projected_shard(type(model).__name__, shard)
        self.model = model
        self.kg_val = kg_val
        self.kg_test = kg_test
        self.shard = shard
        self.is_cuda = next(self.model.parameters()).is_cuda
        self.evaluated = False
        self.thresholds = None
        self.sampler = PositionalNegativeSampler(self.kg_val, kg_test=self.kg_test)

    def _sharded(self):
        """(shard, spec) when the shard splits anything, else (None, None); its argument errors are raised
        here, on every rank, before any collective.  ``spec``: under an EntityShard, the tables the
        per-triple kernel reads (_scoring_spec)."""
        shard = self.shard
        if shard is None or shard.world == 1:
            return None, None
        spec = None
        if isinstance(shard, EntityShard) and shard.local_storage:
            spec = shard_spec(self.model, shard, "TripletClassificationEvaluator", build=self._scoring_spec)
        elif isinstance(shard, EntityShard):
            # the slices are scored by model.scoring_function, which takes kinds the kernel does not
            _check_table(SimpleNamespace(n_ent=self.model.n_ent, ent_lo=0, n_rows=self.model.n_ent), shard)
        return shard, spec

    @staticmethod
    def _scoring_spec(model):
        """ModelSpec over the tables ``model.scoring_function`` hands the per-triple kernel
        (training._param_tensors): RotatE's (cos, sin) planes, TorusE's tables as they are (the kernel
        takes fractional parts), Analogy's planes stacked.  Kinds the kernel does not score raise here."""
        from .training import _kernel_dim, _param_tensors, _training_code
        code = _training_code(model)
        with torch.no_grad():
            e0, e1, r0, r1 = (None if x is None else x.detach() for x in _param_tensors(model, code))
        dim = _kernel_dim(model, code)
        n_ent, n_rel = model.n_ent, model.n_rel
        if code == _lib.ANALOGY:         # stacked (3, n, dim) copies: equally spaced planes
            return ModelSpec(code, dim, n_ent, n_rel, e0[0], e0[1], r0[0], r0[1], ent2=e0[2], rel2=r0[2])
        return ModelSpec(code, dim, n_ent, n_rel, e0, e1, r0, r1)

    def _scores_here(self, heads, tails, relations, batch_size, dev):
        scores = []
        with torch.no_grad():
            for lo in range(0, heads.shape[0], batch_size):
                sl = slice(lo, lo + batch_size)
                scores.append(self.model.scoring_function(heads[sl].to(dev), tails[sl].to(dev),
                                                          relations[sl].to(dev)))
        if not scores:           # a rank whose slice is empty
            return torch.empty(0, dtype=torch.float32, device=dev)
        return torch.cat(scores, dim=0)

    def get_scores(self, heads, tails, relations, batch_size):
        """Scores of the given triplets, computed batch by batch (evaluation.py:478-511)."""
        shard, spec = self._sharded()
        if not self.is_cuda:
            raise _lib.KgeLibraryError("TripletClassificationEvaluator needs the model on a CUDA device")
        dev = next(self.model.parameters()).device
        if shard is None:
            return self._scores_here(heads, tails, relations, batch_size, dev)
        if isinstance(shard, EntityShard) and shard.local_storage:
            h, t, r = (x.to(dev, torch.int64) for x in (heads, tails, relations))
            return score_triples_entity_sharded(spec, h, t, r, shard, default_engine(), batch_size)
        # split by this vector's length, not by a QueryShard's own n
        return _by_query_slices(shard.split(heads.shape[0]), lambda h, t, r, _: [
            self._scores_here(h, t, r, batch_size, dev)], (heads, tails, relations))[0]

    def _negatives(self, b_size, which):
        """``sampler.corrupt_kg``; under a shard, rank 0's draws on every rank (the other ranks add
        zeros into one sum-all-reduce)."""
        nh, nt = self.sampler.corrupt_kg(b_size, self.is_cuda, which=which)
        shard, _ = self._sharded()
        if shard is None:
            return nh, nt
        both = torch.stack([nh, nt]).to(next(self.model.parameters()).device, torch.int64)
        if shard.rank != 0:
            both.zero_()
        both = shard.all_reduce_sum(both).cpu()
        return both[0], both[1]

    def evaluate(self, b_size):
        """Thresholds from the validation graph (evaluation.py:513-541): for relation i the largest
        score among the negatives of its validation facts; relations absent from the validation set
        get the largest negative score overall."""
        r_idx = self.kg_val.relations
        neg_heads, neg_tails = self._negatives(b_size, 'main')
        neg_scores = self.get_scores(neg_heads, neg_tails, r_idx, b_size)
        n_rel = self.kg_val.n_rel
        r_dev = r_idx.to(neg_scores.device)
        per_rel = torch.full((n_rel,), -float("inf"), device=neg_scores.device)
        per_rel = per_rel.scatter_reduce(0, r_dev, neg_scores, reduce="amax", include_self=True)
        present = torch.bincount(r_dev, minlength=n_rel) > 0
        self.thresholds = torch.where(present, per_rel, neg_scores.max()).detach().cpu()
        self.evaluated = True

    def accuracy(self, b_size):
        """Share of test facts scored above, and of their negatives scored below, the threshold
        of their relation (evaluation.py:543-580)."""
        if not self.evaluated:
            self.evaluate(b_size)
        r_idx = self.kg_test.relations
        neg_heads, neg_tails = self._negatives(b_size, 'test')
        scores = self.get_scores(self.kg_test.head_idx, self.kg_test.tail_idx, r_idx, b_size)
        neg_scores = self.get_scores(neg_heads, neg_tails, r_idx, b_size)
        if self.is_cuda:
            self.thresholds = self.thresholds.to(scores.device)
        thr = self.thresholds[r_idx.to(self.thresholds.device)]
        return ((scores > thr).sum().item() + (neg_scores < thr).sum().item()) / (2 * self.kg_test.n_facts)
