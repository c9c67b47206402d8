"""Times the MLP kernel alone on a fixed batch (single sub-module, identity slots): python scripts/mlp_time.py [width] [tiles_per_sm]
MN_B200_PRECISION selects the arithmetic (tc_f16 by default).  Prints ms, TFLOP/s and the SM clock."""
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import torch
import mega_nerf_b200 as M
from mega_nerf_b200 import _cabi as K
from oracle import mn_oracle as O
import cases as Cs
from mega_nerf_b200.synthetic import build_net
from bench import flops_per_row

width = int(sys.argv[1]) if len(sys.argv) > 1 else 256
tps = int(sys.argv[2]) if len(sys.argv) > 2 else 32
dev = torch.device('cuda:0')
spec = O.NerfSpec(layer_dim=width)
net = O.make_net('nerf', spec, seed=3)
n = torch.cuda.get_device_properties(dev).multi_processor_count * 128 * tps
x = Cs.nerf_rows(spec, 4096, 9).repeat(n // 4096 + 1, 1)[:n].contiguous().to(dev)
p = build_net(net, dev)
M.set_precision(os.environ.get('MN_B200_PRECISION', 'tc_f16'))
L, h = K.lib(), K.ctx(dev)
for _ in range(3):
    p(x)
torch.cuda.synchronize()
K.check(L.mn_profile_enable(h, 1), h)
mon = subprocess.Popen(['nvidia-smi', '--query-gpu=clocks.sm,clocks.mem,power.draw,clocks_throttle_reasons.active', '--format=csv,noheader',
                        '-lms', '50'], stdout=subprocess.PIPE, text=True)
reps = 20
for _ in range(reps):
    p(x)
torch.cuda.synchronize()
mon.terminate()
lines = mon.communicate()[0].strip().splitlines()
tot, nl = C.c_double(), C.c_longlong()
K.check(L.mn_profile_read(h, C.byref(tot), C.byref(nl)), h)
ms = tot.value / reps
print(f'width {width} rows {n}: {ms:.3f} ms/launch  {n * flops_per_row(spec) / ms / 1e9:.1f} TFLOP/s   nvidia-smi: {lines[len(lines) // 2] if lines else "-"}')
# correctness of the timed kernel against the fp32 (CUDA-core) path of the same library: an odd and an even tile count
prec = os.environ.get('MN_B200_PRECISION', 'tc_f16')
for rows in (128 * 5 + 17, 128 * 64):
    xs = x[:rows].contiguous()
    M.set_precision(prec)
    got = p(xs).float()
    so = p(xs[:, :3].contiguous(), sigma_only=True).float()
    M.set_precision('fp32')
    ref = p(xs).float()
    err = float((got - ref).abs().max() / ref.abs().max())
    msg = f'rows {rows}: max rel err vs fp32 path {err:.3e}'
    if so is not None:
        rs = p(xs[:, :3].contiguous(), sigma_only=True).float()
        msg += f', sigma_only {float((so - rs).abs().max() / rs.abs().max().clamp_min(1e-9)):.3e}'
    print(msg, 'NaN!' if not torch.isfinite(got).all() else '')
