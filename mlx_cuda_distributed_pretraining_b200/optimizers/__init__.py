from .adamw import AdamW
from .hybrid_optimizer import HybridOptimizer
from .lion import Lion
from .muon import Muon
from .sgd import SGD, SGDEnhanced
from .shampoo import Shampoo, ShampooParams

__all__ = ["AdamW", "Muon", "Shampoo", "ShampooParams", "HybridOptimizer", "Lion", "SGD", "SGDEnhanced"]
