"""The part of ``torchkge.utils`` that sits on the hot path, under the reference's import path
(``from torchkge.utils import MarginLoss`` -> ``from torchkge_b200.utils import MarginLoss``):
the three losses (utils/losses.py), the embedding initialiser (utils/modeling.py:21-28), the
dissimilarity selectors (utils/dissimilarities.py), ``get_bernoulli_probs``
(utils/operations.py:152-179), the batch iterator of the tutorial training loop (``DataLoader``,
utils/data.py:83-151) and the data-redundancy analysis of Akrami et al. (``duplicates``,
``count_triplets``, ``cartesian_product_relations``, utils/data_redundancy.py; on the GPU, see
``torchkge_b200.data_redundancy``).  Dataset downloads, pretrained models and ``Trainer`` (broken at
the reference commit) are outside the scope of this package (DESIGN.md section 7)."""
from .data import DataLoader  # noqa: F401
from .data_redundancy import cartesian_product_relations, count_triplets, duplicates  # noqa: F401
from .losses import BinaryCrossEntropyLoss, LogisticLoss, MarginLoss  # noqa: F401
from .models import (init_embedding, l1_dissimilarity, l1_torus_dissimilarity,  # noqa: F401
                     l2_dissimilarity, l2_torus_dissimilarity)
from .sampling import get_bernoulli_probs  # noqa: F401
