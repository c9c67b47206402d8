"""CPU-only: the host side of the device training batches (mega_nerf_b200/batches.py).  The index batches and the draws from
torch's global generator of `BatchOrder` against the installed torch's own DataLoader iterator, in the two forms
`Runner.train()` builds (runner.py:228-236), after full and partial passes; and which calls of the `DataLoader` binding get
device batches and which get torch's DataLoader."""
import pytest
import torch
from torch.utils.data import DataLoader, Dataset, DistributedSampler

import cases  # noqa: F401  (sys.path setup)
from mega_nerf_b200 import batches as B

pytestmark = pytest.mark.filterwarnings('ignore:.*pin_memory')      # pin_memory=True as the runner passes it, no accelerator here


class Rows(Dataset):
    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n

    def __getitem__(self, idx):
        return idx


def loader_kwargs(ds, batch_size, dist):
    if dist is None:
        return dict(batch_size=batch_size, shuffle=True, num_workers=0, pin_memory=True)
    world, rank = dist
    return dict(batch_size=batch_size // world, sampler=DistributedSampler(ds, world, rank), num_workers=0, pin_memory=True)


def torch_pass(n, batch_size, dist, stop):
    ds = Rows(n)
    out = []
    for k, item in enumerate(DataLoader(ds, **loader_kwargs(ds, batch_size, dist))):
        if k == stop:
            break
        out.append(item.tolist())
    return out


def order_pass(n, batch_size, dist, stop):
    kw = loader_kwargs(Rows(n), batch_size, dist)
    out = []
    for k, idx in enumerate(B.BatchOrder(n, kw['batch_size'], kw.get('sampler'))):
        if k == stop:
            break
        out.append(idx.tolist())
    return out


FORMS = [None, (2, 0), (2, 1), (8, 7)]
LENGTHS = [4096, 4099, 1000]      # a multiple of every batch below, one that is not, one that no world size divides evenly


@pytest.mark.parametrize('dist', FORMS, ids=['shuffle', 'dist2r0', 'dist2r1', 'dist8r7'])
@pytest.mark.parametrize('n', LENGTHS)
@pytest.mark.parametrize('stop', [None, 0, 3])
def test_batches_and_rng_match_torch_dataloader(dist, n, stop):
    batch_size = 256
    want_batches, got_batches, states = [], [], []
    for fn, out in ((torch_pass, want_batches), (order_pass, got_batches)):
        torch.manual_seed(1234)
        for _ in range(2):                                   # two consecutive loaders over the same length
            out.append(fn(n, batch_size, dist, stop))
        states.append(torch.get_rng_state())
    assert got_batches == want_batches
    assert torch.equal(states[0], states[1])
    if stop is None:
        per = batch_size // (1 if dist is None else dist[0])
        assert [len(b) for b in got_batches[0]][:-1] == [per] * (len(got_batches[0]) - 1)
        rows = sum(len(b) for b in got_batches[0])
        assert rows == (n if dist is None else -(-n // dist[0]))
    if dist is not None:
        assert got_batches[0] == got_batches[1]              # the runner never calls set_epoch: same order every time


def test_batch_order_draws_nothing_more_than_the_iterator():
    """The sampler's seed is drawn at the first batch, not when the iterator is made (torch's samplers are generators)."""
    torch.manual_seed(5)
    iter(DataLoader(Rows(100), batch_size=10, shuffle=True, num_workers=0))
    want = torch.get_rng_state()
    torch.manual_seed(5)
    B.BatchOrder(100, 10)
    assert torch.equal(torch.get_rng_state(), want)


def test_sampler_indices_pad_like_distributed_sampler():
    for n, world in ((5, 8), (3, 7), (10, 4), (1, 3)):
        ds = Rows(n)
        for rank in range(world):
            s = DistributedSampler(ds, world, rank, seed=9)
            assert B.sampler_indices(n, s).tolist() == list(iter(s))
            s = DistributedSampler(ds, world, rank, shuffle=False, drop_last=True)
            assert B.sampler_indices(n, s).tolist() == list(iter(s))


class MemoryDataset(Dataset):
    """The reference's MemoryDataset as far as the batches see it (memory_dataset.py:51-63)."""

    def __init__(self, n, rgbs_dtype=torch.float32, img_dtype=torch.int32):
        self._rgbs = torch.rand(n, 3).to(rgbs_dtype)
        self._rays = torch.rand(n, 8)
        self._img_indices = torch.arange(n).to(img_dtype)

    def __len__(self):
        return self._rgbs.shape[0]

    def __getitem__(self, idx):
        return {'rgbs': self._rgbs[idx], 'rays': self._rays[idx], 'img_indices': self._img_indices[idx]}


def test_binding_selects_the_runner_forms():
    ds = MemoryDataset(100)
    dl = B.data_loader(ds, batch_size=32, shuffle=True, num_workers=0, pin_memory=True)
    assert isinstance(dl, B.DeviceBatches) and len(dl) == 4
    dl = B.data_loader(ds, batch_size=16, sampler=DistributedSampler(ds, 8, 3), num_workers=0, pin_memory=True)
    assert isinstance(dl, B.DeviceBatches) and len(dl) == 1
    for kw in (dict(batch_size=32, shuffle=False), dict(batch_size=32, shuffle=True, num_workers=2),
               dict(batch_size=32, shuffle=True, drop_last=True), dict(batch_size=32, shuffle=True, collate_fn=lambda x: x),
               dict(batch_size=32, sampler=torch.utils.data.RandomSampler(ds))):
        assert type(B.data_loader(ds, **kw)) is DataLoader, kw
    assert type(B.data_loader(ds, 32, shuffle=True)) is DataLoader
    assert type(B.data_loader(Rows(100), batch_size=32, shuffle=True)) is DataLoader


@pytest.mark.parametrize('ds', [MemoryDataset(50, rgbs_dtype=torch.float64), MemoryDataset(50, img_dtype=torch.int64)],
                         ids=['rgbs_float64', 'img_int64'])
def test_binding_falls_back_on_other_columns(ds):
    assert type(B.data_loader(ds, batch_size=8, shuffle=True, num_workers=0, pin_memory=True)) is DataLoader


def test_binding_falls_back_on_other_shapes_and_subclasses():
    ds = MemoryDataset(50)
    ds._rays = ds._rays[:, :6].contiguous()
    assert type(B.data_loader(ds, batch_size=8, shuffle=True)) is DataLoader

    class Sub(MemoryDataset):
        pass
    assert type(B.data_loader(Sub(50), batch_size=8, shuffle=True)) is DataLoader
