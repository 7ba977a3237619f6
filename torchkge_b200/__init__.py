"""torchkge_b200 -- H100-native scoring and link-prediction ranking behind the torchkge API.

Drop-in for the hot path of torchkge v0.17.7 (see DESIGN.md / INTEGRATION.md): the classes
below keep the reference's names and signatures; their arithmetic runs in hand-written
sm_90a CUDA kernels reached through the C ABI of ``lib/libkge_b200.so``.
"""
from .exceptions import (NotYetEvaluatedError, NotYetImplementedError, SanityError,  # noqa: F401
                         SizeMismatchError, WrongArgumentsError, WrongDimensionError)
from .data import KnowledgeGraph  # noqa: F401
from .models import (AnalogyModel, ComplExModel, DistMultModel, RESCALModel, RotatEModel,  # noqa: F401
                     TorusEModel, TransDModel, TransEModel, TransHModel)
from .evaluation import (LinkPredictionEvaluator, RelationPredictionEvaluator,  # noqa: F401
                         TripletClassificationEvaluator)
from .inference import EntityInference, RelationInference  # noqa: F401
from .losses import BinaryCrossEntropyLoss, LogisticLoss, MarginLoss  # noqa: F401
from .sampling import (BernoulliNegativeSampler, BernoulliRelationNegativeSampler,  # noqa: F401
                       PositionalNegativeSampler, UniformNegativeSampler)

__version__ = "0.1.0"
