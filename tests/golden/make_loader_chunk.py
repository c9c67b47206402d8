"""Generate tests/golden/loader_chunk_v1.pt: the UNMODIFIED reference's FilesystemDataset._load_chunk_inner (run on the CPU)
on the chunk of tests/test_gpu_zj_loader.py::chunk_dataset, reduced to the pins that test compares.  Needs a checkout of the
reference:    MEGA_NERF_REFERENCE=<path> python tests/golden/make_loader_chunk.py"""
from __future__ import annotations

import os
import sys
import tempfile

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
sys.path.insert(0, os.environ['MEGA_NERF_REFERENCE'])     # a checkout of the reference repository

from ref_shims import install_shims  # noqa: E402
install_shims()
from mega_nerf.datasets.filesystem_dataset import FilesystemDataset  # noqa: E402
import test_gpu_zj_loader as T  # noqa: E402


def main():
    with tempfile.TemporaryDirectory() as d:
        want = FilesystemDataset._load_chunk_inner(T.chunk_dataset(d, torch.device('cpu')))
        pins = T.loader_pins(want)
    torch.save(pins, T.LOADER_GOLDEN_PATH)
    print(f'wrote {T.LOADER_GOLDEN_PATH} ({os.path.getsize(T.LOADER_GOLDEN_PATH) / 1e3:.0f} kB)')


if __name__ == '__main__':
    main()
