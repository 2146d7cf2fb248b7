"""MONAI's metric bookkeeping (monai.metrics.Metric / IterationMetric / Cumulative / RegressionMetric and
do_metric_reduction) as callers of the reference's metrics see it: ``metric(y_pred, y)`` returns the batch's values
[B, ...] and appends them, one entry per batch item, to a buffer; ``aggregate(reduction)`` stacks the buffer and
reduces it with NaNs excluded; ``reset()`` empties it.  Host work on B-element tensors only: no host synchronisation,
so a call can be captured in a CUDA graph."""
from __future__ import annotations

from abc import ABC, abstractmethod

import torch

from ..utils.enums import _StrEnum


class MetricReduction(_StrEnum):
    NONE = "none"
    MEAN = "mean"
    SUM = "sum"
    MEAN_BATCH = "mean_batch"
    SUM_BATCH = "sum_batch"
    MEAN_CHANNEL = "mean_channel"
    SUM_CHANNEL = "sum_channel"


def do_metric_reduction(f: torch.Tensor, reduction: MetricReduction | str = MetricReduction.MEAN):
    """Reduce a [batch, channel, ...] metric tensor, NaNs excluded; returns (f, not_nans), not_nans as float counts.
    MEAN averages over the channel dim first, then over the batch; the *_BATCH and *_CHANNEL modes reduce one dim."""
    nans = torch.isnan(f)
    not_nans = (~nans).float()
    t_zero = torch.zeros(1, device=f.device, dtype=torch.float)
    try:
        reduction = MetricReduction(reduction)
    except ValueError:
        raise ValueError(f"Unsupported reduction: {reduction}, available options are "
                         f"{[m.value for m in MetricReduction]}.") from None
    if reduction == MetricReduction.NONE:
        return f, not_nans
    f[nans] = 0
    if reduction == MetricReduction.MEAN:
        not_nans = not_nans.sum(dim=1)
        f = torch.where(not_nans > 0, f.sum(dim=1).float() / not_nans, t_zero)
        not_nans = (not_nans > 0).float().sum(dim=0)
        f = torch.where(not_nans > 0, f.sum(dim=0).float() / not_nans, t_zero)
    elif reduction == MetricReduction.SUM:
        not_nans = not_nans.sum(dim=[0, 1])
        f = torch.sum(f, dim=[0, 1])
    elif reduction == MetricReduction.MEAN_BATCH:
        not_nans = not_nans.sum(dim=0)
        f = torch.where(not_nans > 0, f.sum(dim=0).float() / not_nans, t_zero)
    elif reduction == MetricReduction.SUM_BATCH:
        not_nans = not_nans.sum(dim=0)
        f = f.sum(dim=0).float()
    elif reduction == MetricReduction.MEAN_CHANNEL:
        not_nans = not_nans.sum(dim=1)
        f = torch.where(not_nans > 0, f.sum(dim=1).float() / not_nans, t_zero)
    elif reduction == MetricReduction.SUM_CHANNEL:
        not_nans = not_nans.sum(dim=1)
        f = f.sum(dim=1).float()
    return f, not_nans


class Metric(ABC):
    @abstractmethod
    def __call__(self, *args, **kwargs):
        raise NotImplementedError


class IterationMetric(Metric):
    """A batch-first tensor is computed as is; a list / tuple of channel-first items one item at a time, the results
    concatenated along the batch."""

    def __call__(self, y_pred, y=None, **kwargs):
        if isinstance(y_pred, (list, tuple)) or isinstance(y, (list, tuple)):
            return self._compute_list(y_pred, y, **kwargs)
        if isinstance(y_pred, torch.Tensor):
            y_ = y.detach() if isinstance(y, torch.Tensor) else None
            return self._compute_tensor(y_pred.detach(), y_, **kwargs)
        raise ValueError("y_pred or y must be a list/tuple of `channel-first` Tensors or a `batch-first` Tensor.")

    def _compute_list(self, y_pred, y=None, **kwargs):
        if y is not None:
            ret = [self._compute_tensor(p.detach().unsqueeze(0), y_.detach().unsqueeze(0), **kwargs)
                   for p, y_ in zip(y_pred, y)]
        else:
            ret = [self._compute_tensor(p_.detach().unsqueeze(0), None, **kwargs) for p_ in y_pred]
        if isinstance(ret[0], torch.Tensor):
            return torch.cat(ret, dim=0)
        if isinstance(ret[0], (list, tuple)) and all(isinstance(i, torch.Tensor) for i in ret[0]):
            return [torch.cat(batch_i, dim=0) for batch_i in zip(*ret)]
        return ret

    @abstractmethod
    def _compute_tensor(self, y_pred, y=None, **kwargs):
        raise NotImplementedError


class Cumulative:
    """A buffer per output of the metric; ``extend`` appends a batch as its items, ``get_buffer`` stacks them."""

    def __init__(self):
        self.reset()

    def reset(self):
        self._buffers = None
        self._synced_tensors = None
        self._synced = False

    def extend(self, *data):
        if self._buffers is None:
            self._buffers = [[] for _ in data]
        for b, d in zip(self._buffers, data):
            d_t = d if isinstance(d, torch.Tensor) else torch.as_tensor(d)
            try:
                b.extend([x[0] for x in torch.split(d_t, 1, dim=0)])
            except (AttributeError, IndexError, RuntimeError) as e:
                raise TypeError(f"{e}. `data` should be a batch-first tensor or a list of channel-first tensors, "
                                f"got {type(d_t)}") from e
        self._synced = False

    def append(self, *data):
        if self._buffers is None:
            self._buffers = [[] for _ in data]
        for b, d in zip(self._buffers, data):
            b.append(d if isinstance(d, torch.Tensor) else torch.as_tensor(d))
        self._synced = False

    def get_buffer(self):
        if not self._synced and self._buffers is not None:
            self._synced_tensors = [torch.stack(b) if b else None for b in self._buffers]
            self._synced = True
        if self._synced_tensors is None:
            return None
        buffers = [x.detach().clone() if isinstance(x, torch.Tensor) else x for x in self._synced_tensors]
        return buffers[0] if len(buffers) == 1 else buffers


class CumulativeIterationMetric(Cumulative, IterationMetric):
    def __call__(self, y_pred, y=None, **kwargs):
        ret = super().__call__(y_pred=y_pred, y=y, **kwargs)
        if isinstance(ret, (tuple, list)):
            self.extend(*ret)
        else:
            self.extend(ret)
        return ret


class RegressionMetric(CumulativeIterationMetric):
    """Checks that y_pred and y have one shape with at least a channel or spatial dim, then ``_compute_metric``."""

    def __init__(self, reduction: MetricReduction | str = MetricReduction.MEAN, get_not_nans: bool = False) -> None:
        super().__init__()
        self.reduction = reduction
        self.get_not_nans = get_not_nans

    def aggregate(self, reduction: MetricReduction | str | None = None):
        data = self.get_buffer()
        if not isinstance(data, torch.Tensor):
            raise ValueError("the data to aggregate must be PyTorch Tensor.")
        f, not_nans = do_metric_reduction(data, reduction or self.reduction)
        return (f, not_nans) if self.get_not_nans else f

    def _check_shape(self, y_pred: torch.Tensor, y: torch.Tensor) -> None:
        if y_pred.shape != y.shape:
            raise ValueError(f"y_pred and y shapes dont match, received y_pred: [{y_pred.shape}] and y: [{y.shape}]")
        if len(y_pred.shape) < 2:
            raise ValueError("either channel or spatial dimensions required, found only batch dimension")

    @abstractmethod
    def _compute_metric(self, y_pred: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        raise NotImplementedError

    def _compute_tensor(self, y_pred, y=None, **kwargs):
        if not isinstance(y_pred, torch.Tensor) or not isinstance(y, torch.Tensor):
            raise ValueError("y_pred and y must be PyTorch Tensor.")
        self._check_shape(y_pred, y)
        return self._compute_metric(y_pred, y)


def require_cuda(*tensors: torch.Tensor) -> None:
    for t in tensors:
        if not t.is_cuda:
            raise RuntimeError("generativemodels_b200.metrics runs on sm_90a (H100) CUDA devices only (input tensor is "
                               "on the CPU and there is no CPU path)")
