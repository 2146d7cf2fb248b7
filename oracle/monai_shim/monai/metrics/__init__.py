from .metric import Cumulative, CumulativeIterationMetric, IterationMetric, Metric  # noqa: F401
from .regression import RegressionMetric  # noqa: F401
from .utils import do_metric_reduction  # noqa: F401
