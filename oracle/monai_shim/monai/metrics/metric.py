"""MONAI's metric base classes (monai/metrics/metric.py), restated for the reference's generative.metrics: a metric
call returns the batch's values and appends them, split per batch item, to a buffer that get_buffer() stacks."""
from abc import ABC, abstractmethod

import torch


class Metric(ABC):
    @abstractmethod
    def __call__(self, *args, **kwargs):
        raise NotImplementedError


class IterationMetric(Metric):
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
            b.extend([x[0] for x in torch.split(d_t, 1, dim=0)])
        self._synced = False

    def append(self, *data):
        if self._buffers is None:
            self._buffers = [[] for _ in data]
        for b, d in zip(self._buffers, data):
            b.append(d if isinstance(d, torch.Tensor) else torch.as_tensor(d))
        self._synced = False

    def _sync(self):
        if self._synced or self._buffers is None:
            return
        self._synced_tensors = [torch.stack(b) if b else None for b in self._buffers]
        self._synced = True

    def get_buffer(self):
        self._sync()
        if self._synced_tensors is None:
            return self._synced_tensors
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
