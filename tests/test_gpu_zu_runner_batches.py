"""GPU: the reference's OWN `Runner.train()` (oracle/_ref/mega_nerf/runner.py, unmodified) on top of `mega_nerf_b200.install()`,
once with the device batches bound over `mega_nerf.runner.DataLoader` and once with torch's DataLoader put back, each in its
own process, both on this library's kernels.  The dataset is the 3-image synthetic directory of test_gpu_zi_runner_dropin,
trained through the reference's own FilesystemDataset (2 parquet chunks of 120 rows, batch 32: 3 full batches and a partial
one per chunk) for 10 iterations across three chunk loads, with a checkpoint at iteration 6, mid-chunk; then resumed from
that checkpoint (the runner skips the batches before its dataset index).  Every batch, every tensor of the saved
checkpoints (weights, optimizer and scaler states, the saved RNG states) and torch's global CPU generator at the end, the
one the DataLoader draws from, must be bit-identical between the two."""
import os
import subprocess
import sys

import pytest
import torch

from test_gpu_zi_runner_dropin import REF, ROOT, make_dataset

pytestmark = pytest.mark.gpu

CHILD = r'''
import os, sys
root, ref, ds, work, mode, ckpt = sys.argv[1:7]
sys.path.insert(0, root); sys.path.insert(0, os.path.join(root, 'tests')); sys.path.insert(0, ref)
import torch
from ref_shims import install_shims
install_shims()
import mega_nerf_b200
mega_nerf_b200.install()
mega_nerf_b200.set_precision('fp32')
mega_nerf_b200.set_train_precision('fp32')
import mega_nerf.runner as RU
from mega_nerf_b200 import batches
assert RU.DataLoader is batches.data_loader
assert RU.render_rays.__module__.startswith('mega_nerf_b200')
if mode == 'torch':
    RU.DataLoader = torch.utils.data.DataLoader
factory, made, seen = RU.DataLoader, [], []


class Recorded:
    def __init__(self, dl):
        self.dl = dl

    def __len__(self):
        return len(self.dl)

    def __iter__(self):
        for item in self.dl:
            seen.append({k: v.to('cuda').cpu() for k, v in item.items()})
            yield item


def recording(*a, **k):
    dl = factory(*a, **k)
    made.append(type(dl).__name__)
    return Recorded(dl)


RU.DataLoader = recording
from mega_nerf.opts import get_opts_base
argv = ['--dataset_path', ds, '--exp_name', os.path.join(work, 'exp' if ckpt == '-' else 'exp_resumed'),
        '--chunk_paths', os.path.join(work, 'chunks'), '--num_chunks', '2', '--batch_size', '32', '--train_iterations', '10',
        '--ckpt_interval', '6', '--no_amp', '--coarse_samples', '16', '--fine_samples', '32', '--near', '0.05', '--far', '1.5',
        '--ray_altitude_range', '-0.6', '0.3', '--val_scale_factor', '1', '--appearance_dim', '0', '--layer_dim', '64',
        '--bg_layer_dim', '64']
if ckpt != '-':
    argv += ['--ckpt_path', ckpt]
parser = get_opts_base()
parser.add_argument('--exp_name', type=str, required=True)
parser.add_argument('--dataset_path', type=str, required=True)
hp = parser.parse_args(argv)
runner = RU.Runner(hp)
assert runner.device.type == 'cuda'
seeds = [torch.cuda.initial_seed()]
# the CUDA generator (depth jitter, density noise) is not the DataLoader's; pin it so that the weights can be compared bit for bit
torch.cuda.manual_seed_all(hp.random_seed)
runner._run_validation = lambda train_index: {}     # the validation metrics need lpips, which this image does not have
runner.train()
seeds.append(torch.cuda.initial_seed())
print('CUDA_SEEDS', seeds)
torch.save({'made': made, 'seen': seen, 'rng': torch.get_rng_state(), 'seeds': seeds},
           os.path.join(work, 'run.pt' if ckpt == '-' else 'resumed.pt'))
print('TRAIN_OK', mode, made)
'''


def run(mode, ds, work, ckpt='-'):
    env = dict(os.environ, TORCH_FORCE_NO_WEIGHTS_ONLY_LOAD='1')     # the runner's checkpoints hold numpy / random states
    r = subprocess.run([sys.executable, '-c', CHILD, ROOT, REF, ds, work, mode, ckpt], capture_output=True, text=True,
                       timeout=900, env=env)
    assert r.returncode == 0 and 'TRAIN_OK' in r.stdout, f'{mode}: rc={r.returncode}\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}'
    return torch.load(os.path.join(work, 'run.pt' if ckpt == '-' else 'resumed.pt'), map_location='cpu', weights_only=False)


def flat(obj, prefix=''):
    """Every leaf of a checkpoint (nested dicts / lists / tuples) by path."""
    if isinstance(obj, dict):
        out = {}
        for k, v in obj.items():
            out.update(flat(v, f'{prefix}/{k}'))
        return out
    if isinstance(obj, (list, tuple)):
        out = {}
        for i, v in enumerate(obj):
            out.update(flat(v, f'{prefix}/{i}'))
        return out
    return {prefix: obj}


def same_leaf(a, b) -> bool:
    if isinstance(a, torch.Tensor):
        return isinstance(b, torch.Tensor) and a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)
    try:
        import numpy as np
        if isinstance(a, np.ndarray):
            return isinstance(b, np.ndarray) and np.array_equal(a, b)
    except ImportError:
        pass
    return a == b


def assert_same_checkpoint(path_a, path_b):
    a = flat(torch.load(path_a, map_location='cpu', weights_only=False))
    b = flat(torch.load(path_b, map_location='cpu', weights_only=False))
    assert set(a) == set(b)
    for ck in (a, b):                                        # the chunk's path: each run has its own chunk directory
        ck['/dataset_state'] = os.path.basename(ck['/dataset_state'])
    bad = [k for k in a if not same_leaf(a[k], b[k])]
    assert not bad, (len(bad), bad[:10])


def assert_same_run(got, want):
    assert len(got['seen']) == len(want['seen']) and len(got['seen']) > 0
    for g, w in zip(got['seen'], want['seen']):
        assert set(g) == set(w)
        for k in w:
            assert g[k].dtype == w[k].dtype and torch.equal(g[k], w[k]), k
    assert torch.equal(got['rng'], want['rng'])             # the generator the DataLoader draws from


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, 'mega_nerf')), reason='oracle/_ref (copy of the reference package, oracle/make_ref.py) not present')
def test_reference_runner_train_with_device_batches(tmp_path):
    ds = str(tmp_path / 'dataset')
    make_dataset(ds)
    works = {m: str(tmp_path / m) for m in ('torch', 'device')}
    for w in works.values():
        os.makedirs(w)
    runs = {m: run(m, ds, w) for m, w in works.items()}
    print('CUDA generator seeds after Runner() / at the end:', {m: r['seeds'] for m, r in runs.items()})
    assert runs['device']['made'] == ['DeviceBatches'] * 3 and runs['torch']['made'] == ['DataLoader'] * 3
    assert len(runs['device']['seen']) == 10
    assert [b['rays'].shape[0] for b in runs['device']['seen']] == [32, 32, 32, 24, 32, 32, 32, 24, 32, 32]
    assert_same_run(runs['device'], runs['torch'])
    models = {m: os.path.join(w, 'exp', '0', 'models') for m, w in works.items()}
    for it in (6, 10):
        assert_same_checkpoint(os.path.join(models['device'], f'{it}.pt'), os.path.join(models['torch'], f'{it}.pt'))
    assert torch.load(os.path.join(models['device'], '6.pt'), map_location='cpu', weights_only=False)['dataset_index'] == 1

    # resume from the checkpoint taken mid-chunk: the runner skips the chunk's first two batches, then trains on
    resumed = {m: run(m, ds, w, os.path.join(models[m], '6.pt')) for m, w in works.items()}
    assert resumed['device']['made'] == ['DeviceBatches'] * 2
    assert [b['rays'].shape[0] for b in resumed['device']['seen']] == [32, 32, 32, 24, 32, 32]      # 2 skipped + 2 + 2
    assert_same_run(resumed['device'], resumed['torch'])
    assert_same_checkpoint(os.path.join(works['device'], 'exp_resumed', '0', 'models', '10.pt'),
                           os.path.join(works['torch'], 'exp_resumed', '0', 'models', '10.pt'))
