"""CPU: the cell test and bit packing of the occupancy render mode (mega_nerf_b200.octree.OccupancyGrid), restated in torch fp32 -
the test the render kernel makes per foreground sample - at the points where it can go wrong: cell faces, the box's faces
(u = 0 inside, u just below 1 inside, u = 1 outside), negative coordinates and NaN; and the grid's cell order, which must be
density_grid's lattice order so that a thresholded density grid packs as it stands."""
import math

import pytest
import torch

import cases  # noqa: F401  (sys.path setup)
from mega_nerf_b200 import octree as T


def _grid(reso, cells, offset=(0.0, 0.0, 0.0), scale=(1.0, 1.0, 1.0)):
    """The grid with exactly the cells (i, j, k) in `cells` occupied."""
    mask = torch.zeros(reso, reso, reso, dtype=torch.bool)
    for c in cells:
        mask[c] = True
    return T.OccupancyGrid.from_mask(mask, offset, scale)


def _cell(u: float, reso: int) -> int:
    """The kernel's cell index of an fp32 u: floorf(u * reso) with the product rounded to fp32."""
    return int(math.floor(float(torch.tensor(u, dtype=torch.float32) * torch.tensor(float(reso), dtype=torch.float32))))


def test_pack_bits_layout():
    g = torch.Generator().manual_seed(0)
    for n in (1, 31, 32, 33, 64, 1000):
        m = torch.rand(n, generator=g) < 0.4
        bits = T.pack_bits(m)
        assert bits.dtype == torch.int32 and bits.numel() == (n + 31) // 32
        for c in range(n):
            assert ((int(bits[c // 32]) >> (c % 32)) & 1) == int(m[c]), (n, c)
        assert torch.equal(T.unpack_bits(bits, n), m)
    # bit 31 set: a negative int32 word
    m = torch.zeros(32, dtype=torch.bool)
    m[31] = True
    assert int(T.pack_bits(m)[0]) == -2 ** 31


@pytest.mark.parametrize('reso', [1, 3, 4, 5, 7, 16])
def test_cell_faces(reso):
    """A point exactly on an inner cell face belongs to the upper cell (floor); u = 0 is cell 0; the largest fp32 below 1 is
    cell reso - 1; u = 1 is outside the box and always queried."""
    below1 = float(torch.nextafter(torch.tensor(1.0), torch.tensor(0.0)))
    for a in range(3):
        for face in range(1, reso):
            u = face / reso
            i = _cell(u, reso)
            assert i in (face - 1, face)        # u = face / reso is itself rounded to fp32
            cell = [0, 0, 0]
            cell[a] = i
            p = torch.zeros(1, 3)
            p[0, a] = u
            # only that cell occupied -> queried; every other cell occupied -> skipped
            assert bool(T.occupancy_queried(p, _grid(reso, [tuple(cell)]))[0])
            others = [(x, y, z) for x in range(reso) for y in range(reso) for z in range(reso) if [x, y, z] != cell]
            assert not bool(T.occupancy_queried(p, _grid(reso, others))[0])
        for u, want in ((0.0, 0), (below1, reso - 1)):
            assert _cell(u, reso) == want
            p = torch.zeros(1, 3)
            p[0, a] = u
            cell = [0, 0, 0]
            cell[a] = want
            assert bool(T.occupancy_queried(p, _grid(reso, [tuple(cell)]))[0])
            assert not bool(T.occupancy_queried(p, _grid(reso, []))[0])
        # u = 1: outside, queried even by an empty grid
        p = torch.zeros(1, 3)
        p[0, a] = 1.0
        assert bool(T.occupancy_queried(p, _grid(reso, []))[0])


def test_fp32_rounding_of_u():
    """u = x * scale + offset is two fp32 roundings, not one fused operation and not float64: pick x, scale, offset where the
    three disagree about the side of a cell face."""
    reso = 4
    scale, offset = 0.3, 0.1
    xs = torch.linspace(-1, 3, 20001, dtype=torch.float32)
    u32 = (xs * torch.tensor(scale, dtype=torch.float32)) + torch.tensor(offset, dtype=torch.float32)
    u64 = xs.double() * float(torch.tensor(scale)) + float(torch.tensor(offset))
    i32 = torch.floor(u32 * reso)
    i64 = torch.floor(u64 * reso)
    differs = ((i32 != i64) & (u32 >= 0) & (u32 < 1)).nonzero().view(-1)
    assert differs.numel() > 0                                   # the restatement is sensitive to the rounding
    for k in differs[:8].tolist():
        x = float(xs[k])
        i = int(i32[k])
        p = torch.tensor([[x, 0.0, 0.0]])
        g = _grid(reso, [(i, 0, 0)], offset=(offset, 0.0, 0.0), scale=(scale, 1.0, 1.0))
        assert bool(T.occupancy_queried(p, g)[0])
        g2 = _grid(reso, [(int(i64[k]), 0, 0)], offset=(offset, 0.0, 0.0), scale=(scale, 1.0, 1.0))
        assert not bool(T.occupancy_queried(p, g2)[0])


def test_negative_and_nan_points_are_queried():
    reso = 4
    empty = _grid(reso, [], offset=(0.5, 0.5, 0.5), scale=(1.0, 1.0, 1.0))
    pts = torch.tensor([[-0.6, 0.0, 0.0], [0.0, -0.5000001, 0.0], [0.0, 0.0, -1e30], [float('nan'), 0.0, 0.0],
                        [0.0, float('nan'), 0.0], [0.0, 0.0, float('inf')], [0.0, 0.0, float('-inf')]])
    assert T.occupancy_queried(pts, empty).all()
    # negative coordinates inside the box (offset 0.5): x = -0.5 is u = 0, cell 0; x = -0.3 is u = 0.2, cell 0
    inside = torch.tensor([[-0.5, -0.5, -0.5], [-0.3, -0.3, -0.3]])
    assert not T.occupancy_queried(inside, empty).any()
    assert T.occupancy_queried(inside, _grid(reso, [(0, 0, 0)], offset=(0.5, 0.5, 0.5))).all()


def test_from_mask_follows_the_density_grid_lattice():
    """The set cells of a random mask over density_grid's rows, located with lattice_points (the reference's grid[mask]),
    are exactly the samples the grid queries among the lattice points; and every lattice point lies in its own cell."""
    reso = 6
    offset = torch.tensor([0.45, 0.52, 0.61])
    scale = torch.tensor([0.37, 0.41, 0.29])
    g = torch.Generator().manual_seed(1)
    mask = torch.rand(reso ** 3, generator=g) < 0.3
    grid = T.OccupancyGrid.from_mask(mask, offset, scale)
    assert grid.reso == reso
    xx, yy, zz = T.lattice_axes(offset, scale, reso)
    lattice = torch.stack(torch.meshgrid(xx, yy, zz, indexing='ij'), -1).reshape(-1, 3)
    q = T.occupancy_queried(lattice, grid)
    assert torch.equal(q, mask)
    occupied = T.lattice_points(mask, offset, scale, reso)
    assert T.occupancy_queried(occupied, grid).all()
    assert occupied.shape[0] == int(mask.sum())
    # the [reso, reso, reso] form indexes [i, j, k]
    grid3 = T.OccupancyGrid.from_mask(mask.view(reso, reso, reso), offset, scale)
    assert torch.equal(grid3.bits, grid.bits)
    assert abs(grid.occupancy() - float(mask.float().mean())) < 1e-6


def test_grid_shape_checks():
    with pytest.raises(ValueError):
        T.OccupancyGrid.from_mask(torch.ones(10, dtype=torch.bool), (0, 0, 0), (1, 1, 1))
    with pytest.raises(ValueError):
        T.OccupancyGrid(torch.zeros(3, dtype=torch.int32), 4, (0, 0, 0), (1, 1, 1))
