"""GPU: training batches gathered on the device (mega_nerf_b200/batches.py, `mn_gather_batch`).  Every batch of the
`DataLoader` binding equals, by torch.equal, the batch the reference's DataLoader (torch's, with the reference datasets'
`__getitem__`) gives moved to the device, in the same order, with torch's global generator left in the same state - on a
parquet chunk loaded through the installed `_load_chunk_inner` and on a MemoryDataset-shaped object; a bad row index is
refused; the fallbacks serve torch's DataLoader."""
import pytest
import torch
from torch.utils.data import DataLoader, Dataset, DistributedSampler

import cases  # noqa: F401
from test_gpu_parity import DEV
from test_gpu_zj_loader import chunk_dataset

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings('ignore:.*pin_memory')]


def B():
    from mega_nerf_b200 import batches
    return batches


class FilesystemDataset(Dataset):
    """The reference's FilesystemDataset as far as the batches see it (filesystem_dataset.py:74-94): the chunk as
    `load_chunk` stores what `_load_chunk_inner` returned."""

    def __init__(self, chunk):
        _, self._loaded_rgbs, self._loaded_rays, self._loaded_img_indices = chunk

    def __len__(self):
        return self._loaded_rgbs.shape[0]

    def __getitem__(self, idx):
        return {'rgbs': self._loaded_rgbs[idx], 'rays': self._loaded_rays[idx], 'img_indices': self._loaded_img_indices[idx]}


class MemoryDataset(Dataset):
    """The reference's MemoryDataset as far as the batches see it (memory_dataset.py:51-63)."""

    def __init__(self, n):
        g = torch.Generator().manual_seed(3)
        self._rgbs = torch.randint(0, 256, (n, 3), generator=g).float() / 255.
        self._rays = torch.randn(n, 8, generator=g)
        self._img_indices = torch.randint(0, 1000, (n,), generator=g, dtype=torch.int32)

    def __len__(self):
        return self._rgbs.shape[0]

    def __getitem__(self, idx):
        return {'rgbs': self._rgbs[idx], 'rays': self._rays[idx], 'img_indices': self._img_indices[idx]}


@pytest.fixture(scope='module')
def fs_dataset(tmp_path_factory):
    from mega_nerf_b200 import loader
    return FilesystemDataset(loader._load_chunk_inner(chunk_dataset(tmp_path_factory.mktemp('chunk'), DEV)))   # 70 000 rows


def runner_kwargs(ds, batch_size, dist):
    if dist is None:
        return dict(batch_size=batch_size, shuffle=True, num_workers=0, pin_memory=True)
    world, rank = dist
    return dict(batch_size=batch_size // world, sampler=DistributedSampler(ds, world, rank), num_workers=0, pin_memory=True)


def passes(make_loader, ds, batch_size, dist, stop):
    """Two consecutive loaders over ds (the second as the runner builds one per chunk), the first stopped after `stop` batches."""
    torch.manual_seed(77)
    out = []
    for p in range(2):
        dl = make_loader(ds, **runner_kwargs(ds, batch_size, dist))
        batches = []
        for k, item in enumerate(dl):
            if p == 0 and k == stop:
                break
            batches.append({key: v.to(DEV, non_blocking=True) for key, v in item.items()})
        out.append((type(dl), len(dl), batches))
    torch.cuda.synchronize()
    return out, torch.get_rng_state()


def check_same(ds, batch_size, dist, stop=None):
    want, want_rng = passes(DataLoader, ds, batch_size, dist, stop)
    got, got_rng = passes(B().data_loader, ds, batch_size, dist, stop)
    assert torch.equal(got_rng, want_rng)
    for (t_want, n_want, b_want), (t_got, n_got, b_got) in zip(want, got):
        assert t_got is B().DeviceBatches and n_got == n_want and len(b_got) == len(b_want)
        for bw, bg in zip(b_want, b_got):
            assert set(bg) == set(bw)
            for k in bw:
                assert bg[k].is_cuda and bg[k].dtype == bw[k].dtype and bg[k].shape == bw[k].shape, k
                assert torch.equal(bg[k], bw[k]), k


FORMS = [None, (2, 0), (2, 1), (8, 7)]
FORM_IDS = ['shuffle', 'dist2r0', 'dist2r1', 'dist8r7']


@pytest.mark.parametrize('dist', FORMS, ids=FORM_IDS)
@pytest.mark.parametrize('batch_size', [1024, 1000])       # 70 000 rows: not a multiple of 1024, a multiple of 1000 (and of 500, 125)
def test_chunk_batches_match_reference_dataloader(fs_dataset, dist, batch_size):
    check_same(fs_dataset, batch_size, dist)


@pytest.mark.parametrize('dist', FORMS, ids=FORM_IDS)
def test_chunk_partial_pass(fs_dataset, dist):
    check_same(fs_dataset, 1024, dist, stop=3)


@pytest.mark.parametrize('dist', FORMS, ids=FORM_IDS)
@pytest.mark.parametrize('n', [8192, 5001])
def test_memory_dataset_batches_match_reference_dataloader(dist, n):
    check_same(MemoryDataset(n), 1024, dist)
    check_same(MemoryDataset(n), 1024, dist, stop=2)


def test_bad_index_is_refused():
    from mega_nerf_b200 import _cabi as K
    ds = MemoryDataset(100)
    cols = [ds._rgbs.to(DEV), ds._rays.to(DEV), ds._img_indices.to(DEV)]
    idx = torch.tensor([3, 100, -1, 99], dtype=torch.int64, device=DEV)
    rgbs, rays, img = B().gather_batch(cols, idx)
    with pytest.raises(RuntimeError, match='index out of range'):
        K.check(K.lib().mn_check_status(K.ctx(DEV), K.stream_of(DEV)), K.ctx(DEV))
    for out, col in ((rgbs, ds._rgbs), (rays, ds._rays), (img, ds._img_indices)):
        assert torch.equal(out[0].cpu(), col[3]) and torch.equal(out[3].cpu(), col[99])
        bits = out[1:3].cpu().view(torch.int32)
        assert bool((bits == -1).all())                      # never read: all one bits
    K.check(K.lib().mn_check_status(K.ctx(DEV), K.stream_of(DEV)), K.ctx(DEV))   # the flag was cleared by the raise


def test_fallbacks_serve_torch_dataloader(monkeypatch):
    ds = MemoryDataset(3000)
    ds._img_indices = ds._img_indices.long()                 # another dtype: the binding returns torch's DataLoader
    assert type(B().data_loader(ds, **runner_kwargs(ds, 1024, None))) is DataLoader
    # an upload that cannot be allocated: the pass is torch's DataLoader's (same batches, same draws)
    ds = MemoryDataset(3000)
    kw = runner_kwargs(ds, 512, None)
    torch.manual_seed(77)
    want = list(DataLoader(ds, **kw))
    want_rng = torch.get_rng_state()

    class Full:
        def to(self, *a, **k):
            raise torch.cuda.OutOfMemoryError('CUDA out of memory (test stand-in)')
    real = B().dataset_columns
    monkeypatch.setattr(B(), 'dataset_columns', lambda d: [Full()] + real(d)[1:])
    torch.manual_seed(77)
    dl = B().data_loader(ds, **kw)
    assert type(dl) is B().DeviceBatches
    it = iter(dl)
    assert isinstance(it, torch.utils.data.dataloader._SingleProcessDataLoaderIter)
    got = list(it)
    assert torch.equal(torch.get_rng_state(), want_rng)
    assert len(got) == len(want) == 6
    for bw, bg in zip(want, got):
        for k in bw:
            assert torch.equal(bg[k], bw[k])


def test_one_launch_per_batch():
    from mega_nerf_b200 import _cabi as K
    ds = MemoryDataset(4096)
    it = iter(B().data_loader(ds, **runner_kwargs(ds, 1024, None)))
    next(it)                                                 # the permutation upload
    before = K.lib().mn_launch_count(K.ctx(DEV))
    next(it)
    assert K.lib().mn_launch_count(K.ctx(DEV)) - before == 1
