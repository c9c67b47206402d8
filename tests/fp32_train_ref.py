"""float64 restatement of fp32 training (the CUDA-core kernels), stage by stage, with a bound on each kernel's deviation.

The fp32 training passes are mlp_simt_kernel<TM, true> (csrc/mn_mlp_simt.cu, the recording forward), mlp_bwd_data_kernel and
mlp_bwd_weight_kernel (csrc/mn_backward.cu).  Every intermediate of theirs is on one of two tapes (TapeLayout, mn_model.cuh;
mn_debug_fp32_train_layout says where): the activation tape (PE, aux, every h_i, F, G, the sigma pre-activation, the rgb head
output, the affine Linear output, the image id) and the gradient tape (every dZ).  Each stage below is seeded from the
kernels' own tape values, so its bound is one rounding step wide and does not grow with depth.  A capture (`cap`) is decoded
per slot, [slots, channels], by tests/test_gpu_zze_train_fp32_stages.py from the GPU, and by tests/test_fp32_train_ref.py
from an fp32 emulation with and without injected bugs.

Rounding points, as the kernels implement them:
  PE / aux    mn_pe_sincos (mn_common.cuh): sincosf(x 2^k), the argument exact (a power of two); CUDA's sincosf is within 2 ulps.
              The xyz / direction columns are the inputs themselves; embedding rows are copied (mn_mlp_simt.cu:147-154) and the
              image id is clamp(int(x[:, -1]), 0, count - 1) (:163-166): all exact.
  Linear      gemm_layer (mn_mlp_simt.cu:13-63): acc = bias, then one fmaf per input column, ascending, PE before h on a skip
              layer (:177-182); ReLU by fmaxf for the trunk and G (:178-182, :219), none for F (:216).
  sigma       acc = sigma_b, fmaf over the last trunk layer, then + noise (:189-195): the stored pre-activation.
  rgb         acc = rgb_b, fmaf over G (or the last trunk layer without dir_a_encoding) (:229-234); the affine head stores that
              Linear output (:240) and transforms it by affine(embedding_a[id]) (:248-266); a colour head stores
              mn_sigmoid (1 / (1 + expf(-v)), :271-272), an SH head the raw coefficients.
  out         x (rgb) and sigma_activation(pre), times the blend weight when blending (:273-276); combine_kernel (mn_route.cu)
              sums a row's slots from 0 in ascending sub-module order.
  heads       GO = grad_out[row] * slot_w (mn_backward.cu:105-107); dsigma = GO_sigma * (softplus'(y = pre - 1) =
              1 / (1 + expf(-y)), 1 above y = 20; or ReLU') (:113-124); d rgb = (GO (1 - s)) s for colour, GO for SH (:126-137).
  affine      dl_q = fmaf chain over c of A[c][q] d_c (:140-184), A = affine(embedding_a[id]) restated; dA atomics into the
              affine and embedding gradients.
  dZ          dgrad_layer (:20-69): acc = 0, one fmaf per output feature of the next Linear, then fmaf(sigma_w, dsigma, .) for
              the last trunk layer (:217), then the mask `tape h > 0` (:63).  dZ_G from W_rgb^T d (:190-199), dZ_F unmasked (:202),
              the last trunk layer without dir_a_encoding from W_rgb^T d + sigma_w dsigma (:219-228).
  embedding   per slot an fmaf chain over the L/2 dZ_G rows times the W_dira embedding columns, atomicAdd to row id (:204-214).
  weights     mlp_bwd_weight_kernel (:274-347): per CTA a sequential fmaf chain over the slots of MN_WG_CHUNK_TILES tiles (bias:
              a sequential sum, added by the k0 == 0 blocks only), then one fp32 atomicAdd per chunk.

Criterion: |k - v| <= beta.  A sequential fmaf chain of n terms from a start value gets beta = (n + 1) u (|start| + sum |a||b|),
u = 2^-24 (the chain's n roundings and the next one).  A weight gradient over a sub-module's slots gets 2 (terms per chunk +
chunks) u sum |dz||x|: each chunk is a chain, the chunks are then added in any order.  Exact checks: padding slots carry dZ = 0
in every channel, a sub-module without slots gets gradients of exactly 0, and a one-hot grad_out (probe) makes every weight
gradient element fp32(dz x) of the probed slot's tape values, bit for bit."""
from __future__ import annotations

import torch

from oracle import mn_oracle as O
from tc_train_ref import U32, Report, app_in_dira, check_output, sigma_act   # noqa: F401  (Report: the callers' table)

MN_BUCKET = 512
MAX_SUB = 64          # MN_MAX_SUB: counters[0..K) counts, [MAX_SUB..MAX_SUB+K] bucket starts, [3 MAX_SUB + 1] slot count
SINCOS_BETA = 4 * U32  # 2 ulps of a value in [-1, 1], twice over


def chain(X, W, start=None):
    """A fmaf chain per output over the columns of X (float64 [n, k]) times W ([out, k], nn.Linear layout), from `start`
    ([out] or None = 0): (v [n, out], beta)."""
    W = W.double()
    v = X @ W.t()
    mag = X.abs() @ W.abs().t()
    if start is not None:
        v = v + start.double()
        mag = mag + start.double().abs()
    return v, (X.shape[1] + 1) * U32 * mag


def pe(x, n_freqs):
    """[x, sin(2^k x), cos(2^k x)]_k in float64 and its bound (0 on the input columns)."""
    v = O.embed(x.double(), n_freqs)
    b = torch.full_like(v, SINCOS_BETA)
    b[:, :x.shape[1]] = 0.0
    return v, b


def image_ids(spec, x):
    return x[:, -1].long().clamp(0, spec.appearance_count - 1)


def affine_T(w, ids):
    """A = affine(embedding_a[id]) as mn_mlp_simt.cu:254-259 chains it: (v [n, 12], beta)."""
    e = w['embedding_a.weight'].double()[ids]
    return chain(e, w['affine.weight'], w['affine.bias'])


def sigmoid_beta(v, b):
    """mn_sigmoid of a value known to within b: 1/4 of b (the slope) plus expf (2 ulps), the add and the divide."""
    s = torch.sigmoid(v)
    return s, 0.25 * b + 8 * U32 * s


# ------------------------------------------------------------------------------------------------------------------------
# captures
# ------------------------------------------------------------------------------------------------------------------------
def ch(cap, name, n=1, off=0):
    """Channels [base + off, base + off + n) of tape block `name` (a_* on the activation tape, g_* on the gradient tape)."""
    t = cap['act'] if name.startswith('a_') else cap['grad']
    b = cap['tl'][name] + off
    return t[:, b:b + n]


def sub_ranges(cap):
    """[(sub-module, first slot, end slot)] in ascending sub-module order."""
    st = cap['starts']
    return [(s, st[i], st[i + 1]) for i, s in enumerate(cap['subs'])]


def restrict(cap, a, b):
    """The capture restricted to slots [a, b)."""
    c = dict(cap)
    for k in ('act', 'grad', 'slot_row'):
        c[k] = cap[k][a:b]
    c['slot_w'] = cap['slot_w'][a:b] if cap['slot_w'] is not None else None
    return c


# ------------------------------------------------------------------------------------------------------------------------
# forward
# ------------------------------------------------------------------------------------------------------------------------
def check_forward(spec: O.NerfSpec, w, c, rep: Report, p=''):
    """The recording forward of one sub-module's slots c (restrict), every stage from the tape values it reads."""
    L, layers, in_xyz = spec.layer_dim, spec.layers, spec.in_xyz
    val = c['slot_row'] >= 0
    if not bool(val.any()):
        return
    x = c['x'][c['slot_row'][val]]
    A = c['act'][val]
    c = dict(c, act=A)
    # ---- encodings
    v, b = pe(x[:, :spec.xyz_dim], spec.pos_xyz_dim)
    rep.f32(p + 'fwd PE', ch(c, 'a_pe', in_xyz), v, b)
    col = 0
    if spec.pos_dir_dim > 0:
        v, b = pe(x[:, -4:-1], spec.pos_dir_dim)
        rep.f32(p + 'fwd dir PE', ch(c, 'a_aux', spec.in_dir), v, b)
        col = spec.in_dir
    if spec.appearance_dim > 0:
        ids = image_ids(spec, x)
        rep.exact(p + 'fwd image id', ch(c, 'a_id')[:, 0], ids.double())
        if app_in_dira(spec):
            rep.exact(p + 'fwd embedding rows', ch(c, 'a_aux', spec.appearance_dim, col), w['embedding_a.weight'].double()[ids])
    # ---- trunk, F, G, each from the tape layer before it
    PE = ch(c, 'a_pe', in_xyz)
    h = [ch(c, 'a_h', L, i * L) for i in range(layers)]
    for i in range(layers):
        X = PE if i == 0 else (torch.cat([PE, h[i - 1]], 1) if i in spec.skip_layers else h[i - 1])
        v, b = chain(X, w[f'xyz_encodings.{i}.0.weight'], w[f'xyz_encodings.{i}.0.bias'])
        rep.f32(p + f'fwd h{i}', h[i], v.clamp(min=0), b)
    H = h[-1]
    if spec.has_dir_a:
        v, b = chain(H, w['xyz_encoding_final.weight'], w['xyz_encoding_final.bias'])
        rep.f32(p + 'fwd F', ch(c, 'a_f', L), v, b)
        FX = torch.cat([ch(c, 'a_f', L), ch(c, 'a_aux', c['tl']['n_aux'])], 1)
        v, b = chain(FX, w['dir_a_encoding.0.weight'], w['dir_a_encoding.0.bias'])
        rep.f32(p + 'fwd G', ch(c, 'a_g', L // 2), v.clamp(min=0), b)
    # ---- heads
    v, b = chain(H, w['sigma.weight'], w['sigma.bias'])
    nz = c['noise'][c['slot_row'][val]].double().view(-1, 1) if c['noise'] is not None else 0.0
    v = v + nz
    rep.f32(p + 'fwd sigma pre-activation', ch(c, 'a_sig'), v, b + U32 * v.abs())
    src = ch(c, 'a_g', L // 2) if spec.has_dir_a else H
    v, b = chain(src, w['rgb.weight'], w['rgb.bias'])
    if spec.affine_appearance and spec.appearance_dim > 0:
        rep.f32(p + 'fwd affine Linear output', ch(c, 'a_lin', 3), v, b)
        r = ch(c, 'a_lin', 3)
        T, bT = affine_T(w, image_ids(spec, x))
        T, bT = T.view(-1, 3, 4), bT.view(-1, 3, 4)
        prod = T[:, :, :3] * r.unsqueeze(1)
        v = prod.sum(-1) + T[:, :, 3]
        b = (bT[:, :, :3] * r.abs().unsqueeze(1)).sum(-1) + bT[:, :, 3] + 4 * U32 * (prod.abs().sum(-1) + T[:, :, 3].abs())
    if spec.rgb_dim == 3:
        v, b = sigmoid_beta(v, b)
    rep.f32(p + 'fwd rgb', ch(c, 'a_rgb', spec.rgb_dim), v, b)


def check_out(spec: O.NerfSpec, cap, rep: Report, p=''):
    """`out` of the recording call from the tape's head values (tc_train_ref.check_output): the rgb columns bit for bit
    through the blend weight and the ascending combine, sigma within sigma_act's bound of the tape's pre-activation."""
    blend = cap['slot_w'] is not None
    pieces = []
    for s, a, b in sub_ranges(cap):
        c = restrict(cap, a, b)
        val = c['slot_row'] >= 0
        if not bool(val.any()):
            continue
        rgb = ch(c, 'a_rgb', spec.rgb_dim)[val]
        sv, sb = sigma_act(spec, ch(c, 'a_sig')[val][:, 0])
        so = dict(v=torch.cat([rgb, sv.view(-1, 1)], 1), beta=torch.cat([torch.zeros_like(rgb), sb.view(-1, 1)], 1),
                  exact=rgb[:, :min(spec.rgb_dim, 3)])
        so = {k: v.cpu() for k, v in so.items()}
        pieces.append((c['slot_row'][val].cpu(), c['slot_w'][val].float().cpu() if blend else None, so))
    check_output(spec, cap['out'].cpu(), pieces, rep, p)
    if spec.rgb_dim > 3 and not blend:
        rows = torch.cat([r for r, _, _ in pieces])
        rgb = torch.cat([so['v'][:, :spec.rgb_dim] for _, _, so in pieces])
        rep.exact(p + 'out SH coefficients = tape (bitwise)', cap['out'].double().cpu()[rows, :spec.rgb_dim], rgb)


# ------------------------------------------------------------------------------------------------------------------------
# backward
# ------------------------------------------------------------------------------------------------------------------------
def head_grads(spec: O.NerfSpec, c, val):
    """GO (fp32, exact as the kernel forms it), (dsigma, beta), (d rgb, beta) of the valid slots of c."""
    rows = c['slot_row'][val]
    go = c['go'][rows].float()
    if c['slot_w'] is not None:
        go = go * c['slot_w'][val].float().view(-1, 1)
    go = go.double()
    pre = ch(c, 'a_sig')[val][:, 0]
    if spec.shifted_softplus:
        y = (pre.float() - 1.0).double()
        d = torch.where(y > 20, torch.ones_like(y), 1 / (1 + torch.exp(-y)))
    else:
        d = (pre > 0).double()
    R = spec.rgb_dim
    ds = go[:, R] * d
    bds = 8 * U32 * ds.abs() if spec.shifted_softplus else torch.zeros_like(ds)
    if R == 3:
        s = ch(c, 'a_rgb', 3)[val]
        dv = (go[:, :3] * (1 - s)) * s
        bdv = 4 * U32 * dv.abs()
    else:
        dv, bdv = go[:, :R], torch.zeros_like(go[:, :R])
    return go, ds, bds, dv, bdv


def masked(name, rep, k, v, b, m):
    """dZ through a ReLU mask m: masked elements must be exactly 0, the others within beta."""
    rep.f32(name, k, v * m, b * m)


def check_backward(spec: O.NerfSpec, w, c, rep: Report, p=''):
    """The data-gradient pass over one sub-module's slots c, each dZ from the tape's dZ of the next Linear."""
    L, layers, in_xyz, R = spec.layer_dim, spec.layers, spec.in_xyz, spec.rgb_dim
    val = c['slot_row'] >= 0
    G = c['grad']
    pad = G[~val]
    rep.exact(p + 'dZ padding slots', pad, torch.zeros_like(pad))
    if not bool(val.any()):
        return
    go, ds, bds, dv, bdv = head_grads(spec, c, val)
    c = dict(c, act=c['act'][val], grad=G[val])
    rep.f32(p + 'bwd dsigma', ch(c, 'g_sig')[:, 0], ds, bds)
    affine = spec.affine_appearance and spec.appearance_dim > 0
    if affine:
        x = c['x'][c['slot_row'][val]]
        T, bT = affine_T(w, image_ids(spec, x))
        T, bT = T.view(-1, 3, 4)[:, :, :3], bT.view(-1, 3, 4)[:, :, :3]
        dl = (T * dv.unsqueeze(-1)).sum(1)
        bdl = (T.abs() * bdv.unsqueeze(-1) + bT * dv.abs().unsqueeze(-1)).sum(1) + 4 * U32 * (T * dv.unsqueeze(-1)).abs().sum(1)
        rep.f32(p + 'bwd affine dl', ch(c, 'g_rgb', 3), dl, bdl)
    else:
        rep.f32(p + 'bwd d rgb', ch(c, 'g_rgb', R), dv, bdv)
    DR, DS = ch(c, 'g_rgb', R), ch(c, 'g_sig')
    H = ch(c, 'a_h', L, (layers - 1) * L)
    Wr = w['rgb.weight'].double()
    sw = w['sigma.weight'].double().view(1, -1)
    if spec.has_dir_a:
        v, b = chain(DR, Wr.t())
        masked(p + 'bwd dZ_G', rep, ch(c, 'g_dira', L // 2), v, b, (ch(c, 'a_g', L // 2) > 0).double())
        Wd = w['dir_a_encoding.0.weight'].double()
        v, b = chain(ch(c, 'g_dira', L // 2), Wd[:, :L].t())
        rep.f32(p + 'bwd dZ_F', ch(c, 'g_final', L), v, b)
        v, b = chain(ch(c, 'g_final', L), w['xyz_encoding_final.weight'].double().t())
    else:
        v, b = chain(DR, Wr.t())
    v = v + DS * sw
    b = b + 2 * U32 * (DS.abs() * sw.abs())
    masked(p + f'bwd dZ_{layers - 1}', rep, ch(c, 'g_z', L, (layers - 1) * L), v, b, (H > 0).double())
    for i in range(layers - 1, 0, -1):
        Wi = w[f'xyz_encodings.{i}.0.weight'].double()
        Wh = Wi[:, in_xyz:] if i in spec.skip_layers else Wi
        v, b = chain(ch(c, 'g_z', L, i * L), Wh.t())
        masked(p + f'bwd dZ_{i - 1}', rep, ch(c, 'g_z', L, (i - 1) * L), v, b, (ch(c, 'a_h', L, (i - 1) * L) > 0).double())


def linear_ops(spec: O.NerfSpec, c):
    """[(state-dict name, dZ [n, N], X [n, K])] of every Linear, from the two tapes (mn_backward.cu:383-400)."""
    L, layers, in_xyz = spec.layer_dim, spec.layers, spec.in_xyz
    PE = ch(c, 'a_pe', in_xyz)
    h = [ch(c, 'a_h', L, i * L) for i in range(layers)]
    ops = []
    for i in range(layers):
        X = PE if i == 0 else (torch.cat([PE, h[i - 1]], 1) if i in spec.skip_layers else h[i - 1])
        ops.append((f'xyz_encodings.{i}.0', ch(c, 'g_z', L, i * L), X))
    ops.append(('sigma', ch(c, 'g_sig'), h[-1]))
    if spec.has_dir_a:
        ops.append(('xyz_encoding_final', ch(c, 'g_final', L), h[-1]))
        ops.append(('dir_a_encoding.0', ch(c, 'g_dira', L // 2), torch.cat([ch(c, 'a_f', L), ch(c, 'a_aux', c['tl']['n_aux'])], 1)))
        ops.append(('rgb', ch(c, 'g_rgb', spec.rgb_dim), ch(c, 'a_g', L // 2)))
    else:
        ops.append(('rgb', ch(c, 'g_rgb', spec.rgb_dim), h[-1]))
    return ops


def check_weight_grads(spec: O.NerfSpec, w, c, grads, rep: Report, p=''):
    """Every parameter gradient of one sub-module per element, from its slots' tape values (padding slots included: their dZ
    is 0, checked by check_backward)."""
    TM, chunk = c['TM'], c['chunk']
    n = c['grad'].shape[0]
    per_chunk = min(n, chunk * TM)
    chunks = -(-n // (chunk * TM))
    k = 2 * (per_chunk + chunks) * U32
    for name, Z, X in linear_ops(spec, c):
        rep.f32(p + f'grad {name}.weight', grads[name + '.weight'], Z.t() @ X, k * (Z.abs().t() @ X.abs()))
        rep.f32(p + f'grad {name}.bias', grads[name + '.bias'], Z.sum(0), k * Z.abs().sum(0))
    if spec.appearance_dim == 0:
        return
    val = c['slot_row'] >= 0
    x = c['x'][c['slot_row'][val]]
    ids = image_ids(spec, x)
    cnt = torch.zeros(spec.appearance_count, 1, dtype=torch.float64, device=x.device).index_add_(
        0, ids, torch.ones(len(ids), 1, dtype=torch.float64, device=x.device))
    ge = grads['embedding_a.weight']
    if app_in_dira(spec):
        L = spec.layer_dim
        We = w['dir_a_encoding.0.weight'].double()[:, L + spec.in_dir:]
        dz = ch(c, 'g_dira', L // 2)[val]
        v = torch.zeros_like(ge, dtype=torch.float64).index_add_(0, ids, dz @ We)
        mag = torch.zeros_like(v).index_add_(0, ids, dz.abs() @ We.abs())
        rep.f32(p + 'grad embedding_a.weight', ge, v, 2 * (L // 2 + cnt) * U32 * mag)
    else:
        go, ds, bds, dv, bdv = head_grads(spec, dict(c), val)
        lin = ch(c, 'a_lin', 3)[val]
        dA = torch.cat([dv.unsqueeze(-1) * lin.unsqueeze(1), dv.unsqueeze(-1)], -1).view(-1, 12)
        bA = torch.cat([bdv.unsqueeze(-1) * lin.abs().unsqueeze(1), bdv.unsqueeze(-1)], -1).view(-1, 12) + U32 * dA.abs()
        m = len(ids)
        rep.f32(p + 'grad affine.bias', grads['affine.bias'], dA.sum(0), bA.sum(0) + 2 * m * U32 * dA.abs().sum(0))
        e = w['embedding_a.weight'].double()[ids]
        rep.f32(p + 'grad affine.weight', grads['affine.weight'], dA.t() @ e, bA.t() @ e.abs() + 2 * (m + 1) * U32 * (dA.abs().t() @ e.abs()))
        Aw = w['affine.weight'].double()                    # [12, app]
        v = torch.zeros_like(ge, dtype=torch.float64).index_add_(0, ids, dA @ Aw)
        mag = torch.zeros_like(v).index_add_(0, ids, dA.abs() @ Aw.abs())
        prop = torch.zeros_like(v).index_add_(0, ids, bA @ Aw.abs())
        rep.f32(p + 'grad embedding_a.weight', ge, v, prop + 2 * (12 + cnt) * U32 * mag)
    unused = torch.ones(spec.appearance_count, dtype=torch.bool, device=ge.device)
    unused[ids] = False
    rep.exact(p + 'grad embedding_a.weight unused ids', ge[unused], torch.zeros_like(ge[unused]))


# ------------------------------------------------------------------------------------------------------------------------
# the whole check of one call
# ------------------------------------------------------------------------------------------------------------------------
def check_call(spec: O.NerfSpec, weights, cap, rep: Report):
    """Every stage of every sub-module that owns slots; exact zeros for the sub-modules that own none (and for the other
    sub-module of a Cascade call); `out` from the tape.  weights / cap['grads']: per sub-module of the model."""
    owned = set()
    multi = len(weights) > 1
    for s, a, b in sub_ranges(cap):
        c = restrict(cap, a, b)
        if b <= a or not bool((c['slot_row'] >= 0).any()):
            continue
        owned.add(s)
        w = {k: v.double() for k, v in weights[s].items()}
        p = f'[{s}] ' if multi else ''
        check_forward(spec, w, c, rep, p)
        check_backward(spec, w, c, rep, p)
        check_weight_grads(spec, w, c, cap['grads'][s], rep, p)
    for s in range(len(weights)):
        if s not in owned:
            for k, v in cap['grads'][s].items():
                rep.exact(f'[{s}] no slots: grad {k}', v, torch.zeros_like(v))
    check_out(spec, cap, rep)


def check_routing(net: O.Net, x, cap, counters, rep: Report):
    """The routed tape against O.route: the slots of each sub-module hold exactly the rows of its mask, padding holds -1,
    slot_w is within 2e-7 of the blend weight, and the bucket starts are the MN_BUCKET-aligned prefix sums of the counts."""
    K = len(net.weights)
    assign, wts = O.route(net, x.cpu())
    mask = (torch.nn.functional.one_hot(assign, K) > 0) if wts is None else wts > 0
    counts = mask.sum(0)
    cnt = counters.long().cpu()
    rep.exact('route counts', cnt[:K].double(), counts.double())
    want = torch.zeros(K + 1, dtype=torch.long)
    want[1:] = torch.cumsum((counts + MN_BUCKET - 1) // MN_BUCKET * MN_BUCKET, 0)
    rep.exact('route bucket starts', cnt[MAX_SUB:MAX_SUB + K + 1].double(), want.double())
    sr = cap['slot_row'].cpu()
    for k in range(K):
        a, n, e = int(want[k]), int(counts[k]), int(want[k + 1])
        got = sr[a:a + n].sort().values
        rows = torch.nonzero(mask[:, k]).view(-1)
        if got.numel() != rows.numel() or not bool((got == rows).all()):
            rep.exact(f'route slot rows of sub-module {k}', torch.ones(1), torch.zeros(1))
        else:
            rep.exact(f'route slot rows of sub-module {k}', got.double(), rows.double())
        rep.exact(f'route padding of sub-module {k}', sr[a + n:e].double(), torch.full((e - a - n,), -1.0, dtype=torch.float64))
        if wts is not None and n:
            rep.f32(f'route slot_w of sub-module {k}', cap['slot_w'][a:a + n].cpu(), wts[sr[a:a + n], k].double(),
                    torch.full((n,), 2e-7, dtype=torch.float64))


def check_probe(spec: O.NerfSpec, cap, row: int, rep: Report, p=''):
    """A grad_out that is nonzero in `row` only: every other slot's dZ is exactly 0, and every weight and bias gradient
    element of a sub-module is fp32(dz x) / dz of the row's slot in it, bit for bit (0 where the row has no slot); the
    embedding gradient is nonzero in the row's image id only."""
    sr = cap['slot_row']
    other = sr != row
    rep.exact(p + 'probe: dZ of the other slots', cap['grad'][other], torch.zeros_like(cap['grad'][other]))
    for s, a, b in sub_ranges(cap):
        c = restrict(cap, a, b)
        hit = torch.nonzero(c['slot_row'] == row).view(-1)
        grads = cap['grads'][s]
        for name, Z, X in linear_ops(spec, c):
            if len(hit):
                j = int(hit[0])
                wv = (Z[j].float().view(-1, 1) * X[j].float().view(1, -1)).double()
                bv = Z[j]
            else:
                wv, bv = torch.zeros_like(grads[name + '.weight']), torch.zeros_like(grads[name + '.bias'])
            rep.exact(p + f'probe: [{s}] grad {name}.weight', grads[name + '.weight'], wv)
            rep.exact(p + f'probe: [{s}] grad {name}.bias', grads[name + '.bias'], bv)
        if app_in_dira(spec):
            ge = grads['embedding_a.weight']
            keep = torch.zeros(ge.shape[0], dtype=torch.bool, device=ge.device)
            if len(hit):
                keep[int(image_ids(spec, cap['x'][row:row + 1])[0])] = True
            rep.exact(p + f'probe: [{s}] grad embedding_a.weight other ids', ge[~keep], torch.zeros_like(ge[~keep]))
