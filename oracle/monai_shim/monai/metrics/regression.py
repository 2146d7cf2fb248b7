"""monai.metrics.regression.RegressionMetric, restated: shape checks, then _compute_metric per batch; aggregate()
reduces the buffer with do_metric_reduction."""
from abc import abstractmethod

import torch

from monai.utils import MetricReduction

from .metric import CumulativeIterationMetric
from .utils import do_metric_reduction


class RegressionMetric(CumulativeIterationMetric):
    def __init__(self, reduction=MetricReduction.MEAN, get_not_nans=False):
        super().__init__()
        self.reduction = reduction
        self.get_not_nans = get_not_nans

    def aggregate(self, reduction=None):
        data = self.get_buffer()
        if not isinstance(data, torch.Tensor):
            raise ValueError("the data to aggregate must be PyTorch Tensor.")
        f, not_nans = do_metric_reduction(data, reduction or self.reduction)
        return (f, not_nans) if self.get_not_nans else f

    def _check_shape(self, y_pred, y):
        if y_pred.shape != y.shape:
            raise ValueError(f"y_pred and y shapes dont match, received y_pred: [{y_pred.shape}] and y: [{y.shape}]")
        if len(y_pred.shape) < 2:
            raise ValueError("either channel or spatial dimensions required, found only batch dimension")

    @abstractmethod
    def _compute_metric(self, y_pred, y):
        raise NotImplementedError

    def _compute_tensor(self, y_pred, y=None, **kwargs):
        if not isinstance(y_pred, torch.Tensor) or not isinstance(y, torch.Tensor):
            raise ValueError("y_pred and y must be PyTorch Tensor.")
        self._check_shape(y_pred, y)
        return self._compute_metric(y_pred, y)
