"""Training batches from a device-resident copy of the loaded chunk: a drop-in for the two DataLoader forms `Runner.train()`
builds (runner.py:228-236) over a `FilesystemDataset` chunk or a `MemoryDataset`,

    DataLoader(dataset, batch_size, shuffle=True, num_workers=0, pin_memory=True)
    DataLoader(dataset, batch_size // world, sampler=DistributedSampler(dataset, world, rank), num_workers=0, pin_memory=True)

The reference assembles each batch on the host, one `__getitem__` per row, then `default_collate`, pinning and a copy to the
device.  Here the chunk's three columns are uploaded once when the iterator starts, the pass's permutation is made with the
same `torch.randperm` call and generator as torch's sampler and uploaded as one tensor, and each batch is one launch of
`mn_gather_batch`.  The batches are bit-identical to the reference's, in the same order, as CUDA tensors with the dtypes and
shapes `default_collate` gives, and torch's global generator is drawn from at the same points as the DataLoader iterator
draws from it.  `install()` binds `data_loader` over `mega_nerf.runner.DataLoader`."""
from __future__ import annotations

import math
from typing import List, Optional, Sequence

import torch
from torch.utils.data import DataLoader, DistributedSampler

from . import _cabi as K

KEYS = ('rgbs', 'rays', 'img_indices')
# (dtype, row width; None = one element per row) of each column, as __getitem__ + default_collate return them
LAYOUT = ((torch.float32, 3), (torch.float32, 8), (torch.int32, None))
# the dataset's attributes holding the three columns (filesystem_dataset.py:75,89-94; memory_dataset.py:51-63).  The two
# classes are recognised by name, so that the reference need not be importable here; a subclass gets torch's DataLoader.
COLUMN_ATTRS = {'FilesystemDataset': ('_loaded_rgbs', '_loaded_rays', '_loaded_img_indices'),
                'MemoryDataset': ('_rgbs', '_rays', '_img_indices')}
_RUNNER_KWARGS = {'batch_size', 'shuffle', 'sampler', 'num_workers', 'pin_memory'}


def sampler_indices(n: int, sampler: Optional[DistributedSampler]) -> torch.Tensor:
    """The rows one pass of the loader's sampler yields, as one int64 tensor, with the sampler's own draws:
    `RandomSampler` without a generator (sampler None) draws a seed from torch's global generator and permutes with a private
    one; `DistributedSampler` permutes under seed + epoch, pads to total_size by repeating the permutation (drop_last False) or
    truncates to it, and keeps every num_replicas-th row from rank."""
    if sampler is None:
        g = torch.Generator()
        g.manual_seed(int(torch.empty((), dtype=torch.int64).random_().item()))
        return torch.randperm(n, generator=g)
    if sampler.shuffle:
        g = torch.Generator()
        g.manual_seed(sampler.seed + sampler.epoch)
        idx = torch.randperm(n, generator=g)
    else:
        idx = torch.arange(n)
    total = sampler.total_size
    if sampler.drop_last:
        idx = idx[:total]
    elif total > n:
        idx = torch.cat([idx, idx.repeat(math.ceil((total - n) / n))[:total - n]])
    return idx[sampler.rank:total:sampler.num_replicas].contiguous()


class BatchOrder:
    """Index batches of one DataLoader pass (batch_size, drop_last False: the last partial batch is kept), drawing from torch's
    global generator where the DataLoader iterator does: its base seed when the iterator is made (`_BaseDataLoaderIter.__init__`),
    the sampler's draws when the first batch is asked for (the batch sampler and the sampler are generators).  With `device`, the
    permutation is uploaded once and the batches are slices of the device copy."""

    def __init__(self, n: int, batch_size: int, sampler: Optional[DistributedSampler] = None,
                 device: Optional[torch.device] = None):
        self.n, self.batch_size, self.sampler, self.device = n, batch_size, sampler, device
        self.indices: Optional[torch.Tensor] = None
        self.pos = 0
        torch.empty((), dtype=torch.int64).random_()

    def __iter__(self):
        return self

    def __next__(self) -> torch.Tensor:
        if self.indices is None:
            idx = sampler_indices(self.n, self.sampler)
            self.indices = idx if self.device is None else idx.to(self.device)
        if self.pos >= self.indices.shape[0]:
            raise StopIteration
        batch = self.indices[self.pos:self.pos + self.batch_size]
        self.pos += self.batch_size
        return batch


def gather_batch(columns: Sequence[torch.Tensor], idx: torch.Tensor) -> List[torch.Tensor]:
    """[c[idx] for c in columns] in one launch: up to three contiguous CUDA columns [n] or [n, w] of 4-byte elements with the
    same n, idx an int64 CUDA tensor [B].  An index outside [0, n) raises at the next `mn_check_status`."""
    if not 1 <= len(columns) <= 3:
        raise ValueError('gather_batch takes one to three columns')
    dev = idx.device
    n = columns[0].shape[0]
    if idx.dtype != torch.int64 or idx.dim() != 1 or not idx.is_contiguous():
        raise ValueError('gather_batch: idx must be a contiguous 1-D int64 tensor')
    args, outs = [], []
    for c in columns:
        if c.device != dev or c.element_size() != 4 or c.dim() not in (1, 2) or c.shape[0] != n or not c.is_contiguous():
            raise ValueError('gather_batch: columns must be contiguous [n] / [n, w] tensors of 4-byte elements on the index device')
        out = torch.empty((idx.shape[0],) + tuple(c.shape[1:]), dtype=c.dtype, device=dev)
        args += [K.ptr(c), c.shape[1] if c.dim() == 2 else 1, K.ptr(out)]
        outs.append(out)
    args += [None, 0, None] * (3 - len(columns))
    h = K.ctx(dev)
    K.check(K.lib().mn_gather_batch(h, K.ptr(idx), idx.shape[0], n, *args, K.stream_of(dev)), h)
    return outs


def dataset_columns(dataset) -> Optional[List[torch.Tensor]]:
    """The (rgbs, rays, img_indices) tensors of a FilesystemDataset's loaded chunk or of a MemoryDataset, or None where the
    dataset is neither or a column has another dtype or shape than the batch kernel takes."""
    attrs = COLUMN_ATTRS.get(type(dataset).__name__)
    if attrs is None:
        return None
    cols = [getattr(dataset, a, None) for a in attrs]
    if not all(isinstance(c, torch.Tensor) for c in cols):
        return None
    n = cols[0].shape[0] if cols[0].dim() > 0 else 0
    for c, (dtype, w) in zip(cols, LAYOUT):
        if c.dtype != dtype or tuple(c.shape) != ((n,) if w is None else (n, w)):
            return None
    return cols if n > 0 else None


class DeviceBatches:
    """What `data_loader` returns for the runner's two forms: iterating it uploads the chunk to the current device and stream
    and yields `{'rgbs', 'rays', 'img_indices'}` batches gathered there.  If the upload cannot be allocated, the pass is
    served by torch's DataLoader instead (same batches, on the host)."""

    def __init__(self, dataset, batch_size: int, sampler: Optional[DistributedSampler], loader_kwargs: dict):
        self.dataset, self.batch_size, self.sampler = dataset, batch_size, sampler
        self._loader_kwargs = loader_kwargs

    def __len__(self) -> int:
        n = len(self.sampler) if self.sampler is not None else len(self.dataset)
        return (n + self.batch_size - 1) // self.batch_size

    def __iter__(self):
        cols = dataset_columns(self.dataset)
        if cols is None:
            raise RuntimeError('the dataset no longer holds a chunk the device batches can serve')
        dev = torch.device('cuda', torch.cuda.current_device())
        try:
            dcols = [c.to(dev).contiguous() for c in cols]
        except torch.cuda.OutOfMemoryError:
            return iter(DataLoader(self.dataset, **self._loader_kwargs))
        return _DeviceBatchIter(dcols, BatchOrder(cols[0].shape[0], self.batch_size, self.sampler, dev))


class _DeviceBatchIter:
    def __init__(self, columns: List[torch.Tensor], order: BatchOrder):
        self.columns, self.order = columns, order

    def __iter__(self):
        return self

    def __next__(self):
        if self.columns is None:
            raise StopIteration
        try:
            idx = next(self.order)
        except StopIteration:
            dev = self.columns[0].device
            self.columns = None                # the chunk's device copy is not kept past the pass
            K.check(K.lib().mn_check_status(K.ctx(dev), K.stream_of(dev)), K.ctx(dev))
            raise
        return dict(zip(KEYS, gather_batch(self.columns, idx)))


def data_loader(dataset, *args, **kwargs):
    """`mega_nerf.runner.DataLoader` after `install()`: device batches (`DeviceBatches`) for a FilesystemDataset or a
    MemoryDataset loaded with the columns the reference makes, in one of the runner's two forms; `torch.utils.data.DataLoader`
    for every other call."""
    sampler = kwargs.get('sampler')
    batch_size = kwargs.get('batch_size', 1)
    runner_form = (not args and set(kwargs) <= _RUNNER_KWARGS and kwargs.get('num_workers', 0) == 0
                   and type(batch_size) is int and batch_size > 0
                   and ((sampler is None and kwargs.get('shuffle') is True)
                        or (type(sampler) is DistributedSampler and not kwargs.get('shuffle'))))
    if runner_form and dataset_columns(dataset) is not None:
        return DeviceBatches(dataset, batch_size, sampler, kwargs)
    return DataLoader(dataset, *args, **kwargs)
