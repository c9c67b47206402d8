"""GPU: tensor-core training (`set_train_precision('tc_f16')`) of the 11- and 12-layer networks at 256 and 512 wide - the
reference's default width and BASELINE configs[3]'s with a deeper trunk (`--layers 11 / 12`, `--skip_layers 4` or `4 8`) - on
the fused engine (tc_mlp_wg_kernel<PP_TRAIN_FWD / PP_DGRAD>, tc_wgrad_kernel), the engine that renders them.

As in tests/test_gpu_zk_train_tc.py and tests/test_gpu_zo_train_512.py the reference is the fp32 CUDA-core training path of the
same library, with the same 16-bit bounds (TC_L2 on the whole gradient vector, TC_TENSOR per tensor).  The boundary tests pin
the engines on either side: 10 layers train on the fused kernel, 13 on the layer-GEMM engine."""
import ctypes as C_
from argparse import Namespace

import pytest
import torch

import cases as C
from mega_nerf_b200 import _cabi as K
from oracle import mn_oracle as O
from test_gpu_parity import DEV, M, product_net, relerr
from test_gpu_zk_train_tc import compare, grads_of, run
from test_gpu_zo_train_512 import many_rows, whole_vector
from test_tp_program import desc as tp_desc

pytestmark = pytest.mark.gpu

HEADS = {
    'rgb_app': dict(),                                  # colour head, direction 4 + appearance 48
    'sh2': dict(pos_dir_dim=0, rgb_dim=27),             # mega-nerf-sh-3's SH degree 2 head
    'bg': dict(xyz_dim=4),                              # background network
}
SKIPS = {'skip4': (4,), 'skip4_8': (4, 8)}
MN_TP_TRAIN_FWD = 1


def deep_spec(width: int, layers: int, skips: str, head: str = 'rgb_app') -> O.NerfSpec:
    return O.NerfSpec(layer_dim=width, layers=layers, skip_layers=SKIPS[skips], **HEADS[head])


def fused_trains(spec: O.NerfSpec) -> bool:
    """Whether the fused kernel has a training program for the shape (the host hook reads the same engine choice as the
    recording call: MN_ERR_UNSUPPORTED for shapes the layer-GEMM engine trains)."""
    d = tp_desc(layer_dim=spec.layer_dim, layers=spec.layers, skips=spec.skip_layers, pos_dir_dim=spec.pos_dir_dim,
                appearance_dim=spec.appearance_dim, rgb_dim=spec.rgb_dim)
    d.xyz_dim = spec.xyz_dim
    tab = (C_.c_uint * (8 * 8192))()
    info = (C_.c_int * 8)()
    return K.lib().mn_debug_tp_program_mode(C_.byref(d), MN_TP_TRAIN_FWD, tab, 8192, info) == 0


def check_single(spec: O.NerfSpec, n_rows: int, tag: str):
    m = M()
    pn = product_net(O.make_net('nerf', spec, seed=31)).requires_grad_(True)
    x = C.nerf_rows(spec, n_rows, 78).to(DEV)
    g = torch.Generator().manual_seed(8)
    cot = (torch.rand(n_rows, spec.rgb_dim + 1, generator=g) - 0.3).to(DEV) * 1e-3
    noise = torch.rand(n_rows, 1, generator=g).to(DEV)
    try:
        m.set_precision('tc_f16')
        with torch.no_grad():
            want = pn(x, sigma_noise=noise)
        out_tc, g_tc = run(pn, x, cot, 'tc_f16', noise)
        assert pn._native().train_on_tensor_cores()
        diff = float((out_tc - want).abs().max())
        assert diff <= 1e-6, diff                                  # the recording forward IS the tc_f16 inference arithmetic
        out_32, g_32 = run(pn, x, cot, 'fp32', noise)
        assert relerr(out_tc, out_32) <= 5e-4
        l2, worst = compare(g_tc, g_32, tag)
        print(f'{tag}: forward vs inference max |diff| {diff:.1e}; tc_f16 training vs fp32: rel L2 {l2:.2e}, worst tensor {worst}')
    finally:
        m.set_train_precision('fp32')


@pytest.mark.parametrize('head', list(HEADS))
@pytest.mark.parametrize('skips', list(SKIPS))
@pytest.mark.parametrize('layers', [11, 12])
@pytest.mark.parametrize('width', [256, 512])
def test_deep_single_network(width, layers, skips, head):
    spec = deep_spec(width, layers, skips, head)
    assert fused_trains(spec)
    check_single(spec, 640, f'{head} {layers}x{width} {skips}')


@pytest.mark.parametrize('width', [256, 512])
def test_deep_single_network_many_tiles(width):
    """More than two tiles per SM: every CTA of the persistent kernels runs several tiles through the shallower ring."""
    check_single(deep_spec(width, 12, 'skip4_8'), many_rows(), f'12x{width} many rows')


@pytest.mark.parametrize('layers,skips', [(11, 'skip4'), (12, 'skip4_8')])
@pytest.mark.parametrize('width', [256, 512])
def test_deep_routed_mega_nerf(width, layers, skips):
    """An 8-sub-module MegaNeRF (2 x 4 grid) at boundary margin 1.15: blended rows reach several sub-modules."""
    m = M()
    spec = deep_spec(width, layers, skips)
    net = O.make_net('mega', spec, seed=7, n_sub=8, centroids=O.grid_centroids(2, 4), boundary_margin=1.15, cluster_2d=True)
    pn = product_net(net).requires_grad_(True)
    x = C.mega_rows(net, 3000, 13).to(DEV)
    g = torch.Generator().manual_seed(6)
    cot = (torch.rand(x.shape[0], 4, generator=g) - 0.5).to(DEV) * 1e-4
    noise = torch.rand(x.shape[0], 1, generator=g).to(DEV)
    try:
        m.set_precision('tc_f16')
        with torch.no_grad():
            want = pn(x, sigma_noise=noise)
        out_tc, g_tc = run(pn, x, cot, 'tc_f16', noise)
        assert pn._native().train_on_tensor_cores()
        assert float((out_tc - want).abs().max()) <= 1e-6
        out_32, g_32 = run(pn, x, cot, 'fp32', noise)
        assert relerr(out_tc, out_32) <= 5e-4
        l2, worst = compare(g_tc, g_32, f'mega8 {layers}x{width}')
        print(f'mega8 {layers}x{width}: tc_f16 training vs fp32: rel L2 {l2:.2e}, worst tensor {worst}')
    finally:
        m.set_train_precision('fp32')


@pytest.mark.parametrize('use_coarse', [True, False])
@pytest.mark.parametrize('width', [256, 512])
def test_deep_cascade(width, use_coarse):
    """A Cascade of two 12-layer networks: each call trains the network it selects."""
    m = M()
    spec = deep_spec(width, 12, 'skip4_8')
    pn = product_net(O.make_net('cascade', spec, seed=5)).requires_grad_(True)
    x = C.nerf_rows(spec, 1000, 44).to(DEV)
    g = torch.Generator().manual_seed(3)
    cot = (torch.rand(x.shape[0], 4, generator=g) - 0.3).to(DEV) * 1e-3

    def step(prec):
        m.set_train_precision(prec)
        pn.zero_grad(set_to_none=True)
        out = pn(use_coarse, x)
        (out * cot).sum().backward()
        torch.cuda.synchronize()
        return out.detach(), grads_of(pn)
    try:
        m.set_precision('tc_f16')
        with torch.no_grad():
            want = pn(use_coarse, x)
        out_tc, g_tc = step('tc_f16')
        assert pn._native().train_on_tensor_cores()
        assert float((out_tc - want).abs().max()) <= 1e-6
        out_32, g_32 = step('fp32')
        assert relerr(out_tc, out_32) <= 5e-4
        l2, worst = compare(g_tc, g_32, f'cascade 12x{width} coarse={use_coarse}')
        print(f'cascade 12x{width} coarse={use_coarse}: tc_f16 training vs fp32: rel L2 {l2:.2e}, worst tensor {worst}')
    finally:
        m.set_train_precision('fp32')


def test_render_rays_12x512_training_step_on_tensor_cores():
    """render_rays in train() mode on an 8-sub-module 12 x 512 MegaNeRF (skips 4 and 8, margin 1.15) with MSE loss: the tc_f16
    step's loss equals the fp32 step's to fp16 accuracy and the gradient vector agrees to TC_L2; 30 Adam steps reduce the loss,
    and one more step then matches the fp32 step at the updated weights, which holds only if the transposed weight images of
    the data-gradient chain were repacked after every opt.step().  Gradients are held to TC_L2 on the whole vector, as for
    the C4 render step of tests/test_gpu_zo_train_512.py."""
    m = M()
    spec = deep_spec(512, 12, 'skip4_8')
    net = O.make_net('mega', spec, seed=0, n_sub=8, centroids=O.grid_centroids(2, 4), boundary_margin=1.15, cluster_2d=True)
    rays = O.synthetic_rays(32, seed=0, far=0.6)
    idx = O.synthetic_indices(32, spec.appearance_count)
    opts = O.RenderOpts(coarse_samples=64, fine_samples=128, perturb=1.0, pos_dir_dim=spec.pos_dir_dim, model_chunk_size=32 * 1024)
    hp = Namespace(**vars(opts))
    target = torch.rand(rays.shape[0], 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    rays_d, idx_d = rays.to(DEV), idx.to(DEV)

    def step(pn, prec, seed):
        m.set_train_precision(prec)
        pn.zero_grad(set_to_none=True)
        torch.manual_seed(seed)
        res, _ = m.render_rays(pn, None, rays_d, idx_d, hp, None, None, False, True, False)
        loss = torch.nn.functional.mse_loss(res['rgb_fine'], target)
        loss.backward()
        return float(loss), grads_of(pn)
    try:
        m.set_precision('tc_f16')
        pn = product_net(net).requires_grad_(True).train()
        l_tc, g_tc = step(pn, 'tc_f16', 11)
        assert pn._native().train_on_tensor_cores()
        l_32, g_32 = step(pn, 'fp32', 11)
        assert abs(l_tc - l_32) <= 2e-3 * abs(l_32), (l_tc, l_32)
        l2, worst = whole_vector(g_tc, g_32, '12x512 render_rays train step')
        print(f'12x512 render_rays step: loss tc {l_tc:.6f} fp32 {l_32:.6f}; grads rel L2 {l2:.2e}, worst {worst}')
        m.set_train_precision('tc_f16')
        opt = torch.optim.Adam(pn.parameters(), lr=5e-4)
        losses = []
        for _ in range(30):
            opt.zero_grad(set_to_none=True)
            res, _ = m.render_rays(pn, None, rays_d, idx_d, hp, None, None, False, True, False)
            loss = torch.nn.functional.mse_loss(res['rgb_fine'], target)
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
        assert all(torch.isfinite(p).all() for p in pn.parameters())
        assert losses[-1] < 0.9 * losses[0], losses
        l_tc, g_tc = step(pn, 'tc_f16', 12)
        l_32, g_32 = step(pn, 'fp32', 12)
        assert abs(l_tc - l_32) <= 2e-3 * abs(l_32), (l_tc, l_32)
        l2, worst = whole_vector(g_tc, g_32, '12x512 render_rays train step after 30 Adam steps')
        print(f'12x512 after Adam: loss tc {l_tc:.6f} fp32 {l_32:.6f}; grads rel L2 {l2:.2e}, worst {worst}')
    finally:
        m.set_train_precision('fp32')


@pytest.mark.parametrize('layers,fused', [(10, True), (13, False)])
@pytest.mark.parametrize('width', [256, 512])
def test_engine_boundary(width, layers, fused):
    """Both sides of the fused kernel's depth range train on the tensor cores: 10 layers on the fused kernel, 13 on the
    layer-GEMM engine (no fused training program), each against the fp32 kernels."""
    spec = deep_spec(width, layers, 'skip4_8')
    assert fused_trains(spec) == fused
    check_single(spec, 640, f'{layers}x{width} ({"fused" if fused else "layer engine"})')
