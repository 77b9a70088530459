"""Model families shipped with the library.  The reference ships exactly one
worked example (data-parallel regression, reference
examples/simple_linear_regression.py); BASELINE.json adds the 4096x4096
data-parallel linear layer."""
from .linear_regression import LinearRegression, make_regression_shard
from .dp_linear import DPLinearModel
from .dp_mlp import DPMLPClassifier, DPMLPModel

__all__ = ["LinearRegression", "make_regression_shard", "DPLinearModel", "DPMLPModel", "DPMLPClassifier"]
