"""``BernoulliNegativeSampler`` with the reference's constructor, attributes and methods
(torchkge/sampling.py:16-138, 226-327).  Corruption runs in a CUDA kernel with a
counter-based generator (Philox4x32-10): same distribution as the reference, not the same
stream -- torch's generators cannot be reproduced from inside a fused kernel (SURVEY.md
section 7, "RNG").
"""
import ctypes

import torch

from . import _lib
from .engine import _ptr, _stream
from .training import fused_loss_step, fused_margin_step, loss_kind_of, refuse_projected_fused_step


def get_bernoulli_probs(kg):
    """dict relation -> tph / (tph + hpt) (torchkge/utils/operations.py:116-179): tph is the
    mean number of tails per (head, relation) pair of the relation, hpt the mean number of
    heads per (relation, tail) pair.  Host-side, one-off; float64 like the pandas original."""
    h, t, r = kg.head_idx.cpu(), kg.tail_idx.cpu(), kg.relations.cpu()
    uhr, c_hr = torch.unique(torch.stack([h, r], 1), dim=0, return_counts=True)
    utr, c_tr = torch.unique(torch.stack([t, r], 1), dim=0, return_counts=True)
    out = {}
    for rel in torch.unique(r).tolist():
        tph = c_hr[uhr[:, 1] == rel].double().mean().item()
        hpt = c_tr[utr[:, 1] == rel].double().mean().item()
        out[rel] = tph / (tph + hpt)
    return out


class NegativeSampler:
    """Interface (torchkge/sampling.py:16-138)."""

    def __init__(self, kg, kg_val=None, kg_test=None, n_neg=1):
        self.kg, self.kg_val, self.kg_test = kg, kg_val, kg_test
        self.n_ent, self.n_facts, self.n_neg = kg.n_ent, kg.n_facts, n_neg
        self.n_facts_val = 0 if kg_val is None else kg_val.n_facts
        self.n_facts_test = 0 if kg_test is None else kg_test.n_facts

    def corrupt_batch(self, heads, tails, relations, n_neg=None):
        raise NotImplementedError

    def corrupt_kg(self, batch_size, use_cuda, which='main'):
        """Corrupt a whole graph with n_neg = 1 (sampling.py:76-138); returns CPU tensors."""
        assert which in ['main', 'train', 'test', 'val']
        kg = {'val': self.kg_val, 'test': self.kg_test}.get(which, self.kg)
        assert kg is not None and kg.n_facts > 0
        if not use_cuda:
            raise _lib.KgeLibraryError("corrupt_kg(use_cuda=False): negative sampling runs on CUDA "
                                       "only in this package")
        nh, nt = [], []
        for lo in range(0, kg.n_facts, batch_size):
            sl = slice(lo, lo + batch_size)
            a, b = self.corrupt_batch(kg.head_idx[sl].cuda(), kg.tail_idx[sl].cuda(),
                                      kg.relations[sl].cuda(), n_neg=1)
            nh.append(a)
            nt.append(b)
        return torch.cat(nh).long().cpu(), torch.cat(nt).long().cpu()


class UniformNegativeSampler(NegativeSampler):
    """Uniform negative sampler (Bordes et al. 2013), torchkge/sampling.py:141-223: head or tail
    with probability 1/2 each, replacement uniform on [1, n_ent) (entity 0 is never drawn, true
    triples are not rejected -- as in the reference).  Same counter-based generator as
    ``BernoulliNegativeSampler``; ``seed`` is an extension.  ``fused_step`` is the fused training step of
    ``BernoulliNegativeSampler`` with every head probability 1/2."""

    def __init__(self, kg, kg_val=None, kg_test=None, n_neg=1, seed=None):
        super().__init__(kg, kg_val, kg_test, n_neg)
        self.seed = int(torch.initial_seed() if seed is None else seed) & 0xFFFFFFFFFFFFFFFF
        self._calls = 0
        self._half = None
        self._halves = None     # (n_rel,) of 1/2 on one device: fused_step's head probabilities

    def corrupt_batch(self, heads, tails, relations=None, n_neg=None):
        if n_neg is None:
            n_neg = self.n_neg
        dev = heads.device
        assert dev == tails.device
        if not heads.is_cuda:
            raise _lib.KgeLibraryError("corrupt_batch needs CUDA index tensors; there is no CPU path")
        b = heads.shape[0]
        if self._half is None or self._half.device != dev:
            self._half = torch.full((1,), 0.5, dtype=torch.float32, device=dev)
        h, t = heads.long().contiguous(), tails.long().contiguous()
        r = torch.zeros(b, dtype=torch.int64, device=dev)   # every fact reads probs[0] = 1/2
        nh = torch.empty(b * n_neg, dtype=torch.int64, device=dev)
        nt = torch.empty(b * n_neg, dtype=torch.int64, device=dev)
        self._calls += 1
        _lib.check(_lib.load().kge_corrupt_batch(_ptr(h), _ptr(t), _ptr(r), b, n_neg, _ptr(self._half),
                                                 self.n_ent, self.seed, self._calls, _ptr(nh), _ptr(nt),
                                                 _stream(dev)), "kge_corrupt_batch")
        return nh, nt

    def _next_offset(self):
        self._calls += 1
        return self._calls

    def fused_step(self, model, heads, tails, relations, margin=None, n_neg=None, *, criterion=None,
                   shard=None):
        """Extension: corruption + ``model(...)`` + the loss in ONE kernel; returns the differentiable scalar
        loss.  Arguments and errors as in ``BernoulliNegativeSampler.fused_step``.  Draws, bit for bit, the
        negatives ``corrupt_batch`` would draw at the same call count: the Bernoulli step with every
        probability 1/2."""
        n = max(int(self.kg.n_rel), int(getattr(model, "n_rel", 0)))   # every relation id the batch may hold
        dev = heads.device
        if self._halves is None or self._halves.device != dev or self._halves.shape[0] != n:
            self._halves = torch.full((n,), 0.5, dtype=torch.float32, device=dev)
        return _sampler_fused_step(self, model, heads, tails, relations, margin, n_neg, criterion, shard,
                                   self._halves)


class BernoulliNegativeSampler(NegativeSampler):
    """Bernoulli negative sampler (Wang et al. 2014), torchkge/sampling.py:226-327.

    Attributes
    ----------
    bern_probs: torch.FloatTensor (n_rel,) -- probability of corrupting the HEAD per relation
        (0.5 for relations absent from ``kg``).
    seed: int -- key of the counter-based generator (extension; defaults to torch's seed).
    """

    def __init__(self, kg, kg_val=None, kg_test=None, n_neg=1, seed=None):
        super().__init__(kg, kg_val, kg_test, n_neg)
        self.bern_probs = self.evaluate_probabilities()
        self.seed = int(torch.initial_seed() if seed is None else seed) & 0xFFFFFFFFFFFFFFFF
        self._calls = 0

    def evaluate_probabilities(self):
        probs = get_bernoulli_probs(self.kg)
        return torch.tensor([probs.get(i, 0.5) for i in range(self.kg.n_rel)]).float()

    def _next_offset(self):
        self._calls += 1
        return self._calls

    def corrupt_batch(self, heads, tails, relations, n_neg=None):
        """(neg_heads, neg_tails), int64, on ``heads.device``, laid out as n_neg blocks of the
        batch; entity 0 is never drawn and true triples are not rejected, as in the reference."""
        if n_neg is None:
            n_neg = self.n_neg
        dev = heads.device
        assert dev == tails.device
        if not heads.is_cuda:
            raise _lib.KgeLibraryError("corrupt_batch needs CUDA index tensors; there is no CPU path")
        b = heads.shape[0]
        self.bern_probs = self.bern_probs.to(dev)
        h, t, r = (x.long().contiguous() for x in (heads, tails, relations))
        nh = torch.empty(b * n_neg, dtype=torch.int64, device=dev)
        nt = torch.empty(b * n_neg, dtype=torch.int64, device=dev)
        _lib.check(_lib.load().kge_corrupt_batch(_ptr(h), _ptr(t), _ptr(r), b, n_neg,
                                                 _ptr(self.bern_probs), self.n_ent, self.seed,
                                                 self._next_offset(), _ptr(nh), _ptr(nt), _stream(dev)),
                   "kge_corrupt_batch")
        return nh, nt

    def fused_step(self, model, heads, tails, relations, margin=None, n_neg=None, *, criterion=None,
                   shard=None):
        """Extension: corruption + ``model(...)`` + the loss in ONE kernel; returns the differentiable
        scalar loss.  Draws the negatives ``corrupt_batch`` would draw at the same call count.

        Give exactly one of ``margin`` (``MarginLoss(margin)``) and ``criterion`` (a ``MarginLoss``,
        ``LogisticLoss`` or ``BinaryCrossEntropyLoss``; see ``training.fused_loss_step``).

        shard: ``EntityShard(local_storage=True)`` for a model holding only its entity rows (see
        ``training.fused_margin_step``); every rank uses a sampler with the same seed and call count,
        built on the whole graph, and passes the same batch."""
        self.bern_probs = self.bern_probs.to(heads.device)
        return _sampler_fused_step(self, model, heads, tails, relations, margin, n_neg, criterion, shard,
                                   self.bern_probs)


def _sampler_fused_step(sampler, model, heads, tails, relations, margin, n_neg, criterion, shard, probs,
                        rel_share=None, positional=None):
    """fused_step of the samplers: their argument checks, then the fused step at the sampler's next call count
    with head probabilities ``probs`` (rel_share: the relation-corrupting step; positional: the positional
    step's CSR)."""
    refuse_projected_fused_step(model)
    if (margin is None) == (criterion is None):
        raise ValueError("fused_step takes exactly one of margin and criterion")
    if criterion is not None:
        loss_kind_of(criterion)       # an unsupported criterion raises before the call count moves
    if n_neg is None:
        n_neg = sampler.n_neg
    if shard is not None and getattr(shard, "n_ent", sampler.n_ent) != sampler.n_ent:
        raise ValueError("the sampler draws on %d entities, the shard partitions %d"
                         % (sampler.n_ent, shard.n_ent))
    if positional is not None and shard is None and int(model.n_ent) != sampler.n_ent:
        # the kernel indexes the model's table with the sampler's entity ids
        raise ValueError("the sampler draws on %d entities, the model has %d" % (sampler.n_ent, model.n_ent))
    if criterion is not None:
        return fused_loss_step(model, heads, tails, relations, criterion, n_neg=n_neg, bern_probs=probs,
                               seed=sampler.seed, offset=sampler._next_offset(), shard=shard,
                               rel_share=rel_share, positional=positional)
    return fused_margin_step(model, heads, tails, relations, margin, n_neg=n_neg, bern_probs=probs,
                             seed=sampler.seed, offset=sampler._next_offset(), shard=shard, rel_share=rel_share,
                             positional=positional)


class BernoulliRelationNegativeSampler(NegativeSampler):
    """Bernoulli sampler that also corrupts relations, torchkge/sampling.py:507-553: with probability
    ``rel_share`` a negative replaces an entity -- the head with probability ``bern_probs[r]``, else the
    tail, uniform on [1, n_ent) -- and otherwise its relation, uniform on [1, n_rel).  Exactly one
    position changes; entity 0 and relation 0 are never drawn and true triples are not rejected, as in the
    reference.  Use with ``model(h, t, r, nh, nt, nr)``.

    Draws come from the counter-based generator of ``BernoulliNegativeSampler`` (kge_corrupt_batch_rel):
    with the same seed and call count, ``rel_share = 1`` gives that sampler's negatives.

    Attributes
    ----------
    bern_probs: torch.FloatTensor (n_rel,) -- probability of corrupting the HEAD of an entity negative
        (0.5 for relations absent from ``kg``).
    rel_share: float -- probability that a negative replaces an entity rather than the relation.
    seed: int -- key of the counter-based generator (extension; defaults to torch's seed).
    """

    def __init__(self, kg, kg_val=None, kg_test=None, n_neg=1, rel_share=.33, seed=None):
        super().__init__(kg, kg_val, kg_test, n_neg)
        self.n_rel = kg.n_rel
        rel_share = float(rel_share)
        if not 0.0 <= rel_share <= 1.0:
            raise ValueError("rel_share must lie in [0, 1], got %r" % (rel_share,))
        if self.n_rel < 2 and rel_share < 1.0:
            raise ValueError("relation corruption draws from [1, n_rel) and needs n_rel >= 2 (n_rel = %d)"
                             % self.n_rel)
        self.rel_share = rel_share
        self.bern_probs = self.evaluate_probabilities()
        self.seed = int(torch.initial_seed() if seed is None else seed) & 0xFFFFFFFFFFFFFFFF
        self._calls = 0

    evaluate_probabilities = BernoulliNegativeSampler.evaluate_probabilities
    _next_offset = BernoulliNegativeSampler._next_offset

    def corrupt_batch(self, heads, tails, relations, n_neg=None):
        """(neg_heads, neg_tails, neg_rels), int64, on ``heads.device``: ONE negative per fact, as in the
        reference (``n_neg`` is ignored: ``Model.forward`` cannot pair blocks of relations with an
        unrepeated positive)."""
        dev = heads.device
        assert dev == tails.device
        if not heads.is_cuda:
            raise _lib.KgeLibraryError("corrupt_batch needs CUDA index tensors; there is no CPU path")
        b = heads.shape[0]
        self.bern_probs = self.bern_probs.to(dev)
        h, t, r = (x.to(dev).long().contiguous() for x in (heads, tails, relations))
        nh, nt, nr = (torch.empty(b, dtype=torch.int64, device=dev) for _ in range(3))
        _lib.check(_lib.load().kge_corrupt_batch_rel(_ptr(h), _ptr(t), _ptr(r), b, 1, _ptr(self.bern_probs),
                                                     self.n_ent, self.n_rel, self.rel_share, self.seed,
                                                     self._next_offset(), _ptr(nh), _ptr(nt), _ptr(nr),
                                                     _stream(dev)), "kge_corrupt_batch_rel")
        return nh, nt, nr

    def corrupt_kg(self, batch_size, use_cuda, which='main'):
        """Corrupt a whole graph (one negative per fact): (neg_heads, neg_tails, neg_rels), CPU tensors.
        The reference inherits a two-value version that fails for this sampler."""
        assert which in ['main', 'train', 'test', 'val']
        kg = {'val': self.kg_val, 'test': self.kg_test}.get(which, self.kg)
        assert kg is not None and kg.n_facts > 0
        if not use_cuda:
            raise _lib.KgeLibraryError("corrupt_kg(use_cuda=False): negative sampling runs on CUDA "
                                       "only in this package")
        out = ([], [], [])
        for lo in range(0, kg.n_facts, batch_size):
            sl = slice(lo, lo + batch_size)
            for acc, x in zip(out, self.corrupt_batch(kg.head_idx[sl].cuda(), kg.tail_idx[sl].cuda(),
                                                      kg.relations[sl].cuda())):
                acc.append(x)
        return tuple(torch.cat(x).long().cpu() for x in out)

    def fused_step(self, model, heads, tails, relations, margin=None, n_neg=None, *, criterion=None,
                   shard=None):
        """Extension: corruption + ``model(h, t, r, nh, nt, nr)`` + the loss in ONE kernel; returns the
        differentiable scalar loss.  Arguments and errors as in ``BernoulliNegativeSampler.fused_step``.

        n_neg (extension) >= 1 negatives per fact, drawn as n_neg blocks of the batch; block 0 is exactly
        what ``corrupt_batch`` draws at the same call count.  With ``shard``, the rank holding a positive's
        head scores its relation negatives."""
        self.bern_probs = self.bern_probs.to(heads.device)
        return _sampler_fused_step(self, model, heads, tails, relations, margin, n_neg, criterion, shard,
                                   self.bern_probs, rel_share=self.rel_share)


class PositionalNegativeSampler(BernoulliNegativeSampler):
    """Positional negative sampler (Socher et al. 2013), torchkge/sampling.py:330-503: head or tail
    by Bernoulli(p_r) as in Wang et al. 2014; the replacement is drawn uniformly among the entities
    that occupy the same position in some fact of the same relation (in ``kg`` and ``kg_val``, not
    ``kg_test``); a relation never seen gets a uniform entity.  Always one negative per fact.

    The reference walks Python lists fact by fact (sampling.py:476-501); here the candidate sets are
    two CSR arrays on the device and a batch is three gathers.  Draws come from a ``torch.Generator``
    on the batch's device (seeded by ``seed``): same law as the reference, not the same stream.

    ``fused_step`` (extension) draws the same law inside the fused training step, from the counter-based
    generator of ``BernoulliNegativeSampler`` keyed by ``seed`` -- so not the stream ``corrupt_batch`` draws,
    whose ``torch.Generator`` (and with it ``TripletClassificationEvaluator``'s default negatives) is unchanged.

    Attributes: ``possible_heads`` / ``possible_tails`` (dict relation -> sorted list),
    ``n_poss_heads`` / ``n_poss_tails`` (LongTensor (n_rel,)), as in the reference.
    """

    def __init__(self, kg, kg_val=None, kg_test=None, seed=None):
        super().__init__(kg, kg_val, kg_test, 1, seed=seed)
        graphs = [kg] + ([kg_val] if kg_val is not None and kg_val.n_facts > 0 else [])
        h = torch.cat([g.head_idx for g in graphs]).long()
        t = torch.cat([g.tail_idx for g in graphs]).long()
        r = torch.cat([g.relations for g in graphs]).long()
        self._csr = {}
        for name, e in (("heads", h), ("tails", t)):
            key = torch.unique(r * self.n_ent + e)               # sorted by (relation, entity)
            rel_of, ent_of = torch.div(key, self.n_ent, rounding_mode="floor"), key % self.n_ent
            counts = torch.bincount(rel_of, minlength=kg.n_rel)
            offs = torch.zeros(kg.n_rel + 1, dtype=torch.int64)
            offs[1:] = torch.cumsum(counts, 0)
            self._csr[name] = (offs, ent_of, counts)
        self.n_poss_heads, self.n_poss_tails = self._csr["heads"][2], self._csr["tails"][2]
        self._dev = {}
        self._gen = {}

    def _lists(self, name):
        offs, ents, _ = self._csr[name]
        return {rel: ents[offs[rel]:offs[rel + 1]].tolist() for rel in range(self.kg.n_rel)}

    @property
    def possible_heads(self):
        return self._lists("heads")

    @property
    def possible_tails(self):
        return self._lists("tails")

    def _on(self, dev):
        if dev not in self._dev:
            self._dev[dev] = {k: tuple(x.to(dev) for x in v) for k, v in self._csr.items()}
            g = torch.Generator(device=dev)
            g.manual_seed(self.seed & 0x7FFFFFFFFFFFFFFF)
            self._gen[dev] = g
        return self._dev[dev], self._gen[dev]

    def corrupt_batch(self, heads, tails, relations, n_neg=None):
        dev = heads.device
        assert dev == tails.device
        if not heads.is_cuda:
            raise _lib.KgeLibraryError("corrupt_batch needs CUDA index tensors; there is no CPU path")
        csr, gen = self._on(dev)
        self.bern_probs = self.bern_probs.to(dev)
        rel = relations.long()
        b = heads.shape[0]
        head_mask = torch.rand(b, device=dev, generator=gen) < self.bern_probs[rel]
        u = torch.rand(b, device=dev, generator=gen)
        any_ent = torch.randint(0, self.n_ent, (b,), device=dev, generator=gen)
        out = []
        for name, orig, mask in (("heads", heads.long(), head_mask), ("tails", tails.long(), ~head_mask)):
            offs, ents, counts = csr[name]
            n_poss = counts[rel]
            choice = (n_poss.float() * u).floor().long().clamp_(max=(n_poss - 1).clamp(min=0))
            pos = (offs[rel] + choice).clamp_(max=max(ents.numel() - 1, 0))
            drawn = ents[pos] if ents.numel() > 0 else any_ent
            drawn = torch.where(n_poss > 0, drawn, any_ent)
            out.append(torch.where(mask, drawn, orig))
        return out[0], out[1]

    def fused_step(self, model, heads, tails, relations, margin=None, n_neg=None, *, criterion=None,
                   shard=None):
        """Extension: positional corruption + ``model(...)`` + the loss in ONE kernel; returns the differentiable
        scalar loss.  Arguments and errors as in ``BernoulliNegativeSampler.fused_step``; the model must have the
        sampler's ``n_ent`` entities (with ``shard``: the shard must partition them).

        Each negative replaces the head with probability ``bern_probs[r]``, else the tail, by an entity drawn
        uniformly from ``possible_heads[r]`` / ``possible_tails[r]``, or from [0, n_ent) when that list is empty,
        as in ``corrupt_batch`` -- the same law, drawn by the counter-based generator at the sampler's next call
        count rather than from ``corrupt_batch``'s stream.  n_neg (extension) >= 1 negatives per fact, as n_neg
        blocks of the batch.  With ``shard`` every rank holds the whole candidate CSR; the rank holding the
        drawn entity scores a negative."""
        csr, _ = self._on(heads.device)
        positional = (csr["heads"][0], csr["heads"][1], csr["tails"][0], csr["tails"][1])
        self.bern_probs = self.bern_probs.to(heads.device)
        return _sampler_fused_step(self, model, heads, tails, relations, margin, n_neg, criterion, shard,
                                   self.bern_probs, positional=positional)
