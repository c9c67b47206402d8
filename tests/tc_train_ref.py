"""float64 restatement of tensor-core training (precision 'tc_f16'), stage by stage, with a bound on each kernel's deviation.

Two users:
  wide_tc_chain      the whole chain from rows to parameter gradients (fp16 rounding as `rnd`, or none), compared with the
                     oracle's autograd by tests/test_backward_wide_algorithm.py and tests/test_backward_512_algorithm.py.
  check_stages       every stage seeded from the kernels' own intermediates (encoder tiles, activation records, fp32 head
                     blocks, head-gradient blocks, dZ images, embedding sums), so no bound propagates through depth: each
                     stage is one rounding step away from its inputs.  tests/test_gpu_zzc_train_tc_stages.py feeds it what the
                     GPU wrote; tests/test_tc_train_ref.py an fp32 emulation, with and without injected bugs.
  check_forward      its forward half alone (check_backward the rest), for every network with a tensor-core forward: also
                     the 64..192-wide fused plans, the affine colour head and the rgb head that reads the trunk directly.
  check_output       output assembly: `out` from the head block and the head input image (slot_outputs), through the blend
                     weight and combine_kernel's sum.  tests/test_gpu_zzd_infer_tc.py feeds both the recording forward of a
                     tc_f16 inference call (mn_debug_tc_forward_record), whose `out` equals that call's bit for bit.

Rounding points, as the kernels implement them:
  encoder     tc_encode_kernel / tc_encode_fast_kernel (mn_mlp_tc.cu): x, sin(2^k x), cos(2^k x) in fp32 (sincosf, or the
              fast encoder's pe_band: sincosf every fourth band, double-angle recurrences between), then fp16.  Direction PE the
              same; embedding rows are the fp32 weights rounded to fp16.  PE_BETA bounds the fp32 error of both encoders.
  trunk/F/G   fp16 X times fp16 W (the pack rounds fp32 weights to fp16), fp32 accumulation, + fp32 bias, ReLU (none for F =
              xyz_encoding_final), fp16 (mn_mlp_wg.cuh epilogue, mn_layer_gemm.cuh epilogue).
  sigma       fused engine: sum of the fp32 post-ReLU values of the last trunk layer times fp32 sigma_w, before they are
              rounded (mn_mlp_wg.cuh, sacc_a / sacc_b); those values are not on the tape, so beta adds sum |w_sigma| half-ulp16(h).
              Layer engine: tc_layer_head_kernel sums the fp16 tape image times fp32 sigma_w (mn_layer_gemm.cuh).  Then
              + sigma_b + noise, stored as the fp32 pre-activation.
  rgb         fused engine: an MMA, fp16 G times fp16 W_rgb; layer engine: fp16 G times fp32 W_rgb on CUDA cores (the last
              trunk image instead of G without dir_a_encoding).  Colour heads store sigmoid(pre) in the fp32 head block; the
              affine head (tc_emit_rgb) transforms pre by affine(embedding_a[id]) first and stores only to `out`.
  out         tc_emit_rgb / the sigma epilogue: x (rgb) and sigma_activation(pre) (mn_softplus_shifted or fmaxf), times the
              slot's blend weight when blending; combine_kernel sums a row's slots in fp32, ascending sub-module order.
  backward    S = 2^(10 - ceil(log2 max|grad_out|)) (tc_grad_scale_kernel).  Head stage in fp32 (tc_head_grad): d = (g w (1 -
              c)) c for colour, g w for SH; dsigma = g_sigma w ReLU'(pre) or softplus'(pre - 1).  dZ_G = mask(G > 0)
              (sum_c W_rgb[c] d[c]) in fp32 (tc_rgb_dgrad8), times S, fp16.  Data-gradient GEMMs: fp16 dZ times fp16 W, fp32
              accumulation, then fmaf(S dsigma, sigma_w, .) for the last trunk layer, then the mask `tape image > 0` (so a
              positive pre-activation that rounded to fp16 zero is masked), fp16.  Weight gradients dZ^T X / S (tc_wgrad_kernel,
              bias through an all-ones operand); heads from the fp32 head-gradient blocks times fp16 tape images
              (tc_heads_wgrad_kernel); embedding from per-image sums of the unscaled fp32 dZ_G rows (tc_emb_sums8) times the
              fp32 W_dira embedding columns (tc_emb_grad_kernel).

Criterion: an fp16 image element k passes when h16(op(v - beta)) <= k <= h16(op(v + beta)), op being the stage's monotone
post-operation (ReLU, the mask, S); an fp32 value when |k - v| <= beta.  A dot product of n terms gets beta = C_DOT n 2^-24
sum |a||b|: wgmma's fp32 accumulation is not round-to-nearest per add (it may truncate: 2 units per add), and fp32 atomics
add in any order, both covered by C_DOT = 2 with the n u sum|a||b| worst-case bound of any summation order."""
from __future__ import annotations

import math

import torch

from oracle import mn_oracle as O

U32 = 2.0 ** -24
C_DOT = 2.0
# fp32 error of an encoder feature (absolute; features lie in [-1, 1] or are the inputs themselves).  sincosf is within 2 ulps;
# pe_band's three doublings grow the error of the band they start from by at most 6x each (|ds'| <= 2(|ds| + |dc|), |dc'| <=
# 4|ds|), and tests/test_tc_train_ref.py measures the fp32 recurrence at 1.4e-6 (the H100 encoder at 1.3e-6).
PE_BETA = 8e-6


def h16(t):
    """fp16 rounding, in the tensor's own dtype."""
    return t.half().to(t.dtype)


def half_ulp16(t):
    """half an fp16 ulp at |t| (the largest rounding error of a value that rounds to t), subnormal spacing below 2^-14."""
    a = t.abs().double()
    _, e = torch.frexp(a)
    return torch.where(a > 0, torch.ldexp(torch.ones_like(a), e - 12), torch.zeros_like(a)).clamp(min=2.0 ** -25)


def grad_scale(cot):
    m = float(cot.abs().max()) if cot.numel() else 0.0
    return 2.0 ** (10 - math.ceil(math.log2(m))) if 0 < m < 3e38 else 1.0


def errors(got, want):
    num = den = 0.0
    worst = ('', 0.0)
    for k, v in want.items():
        num += float((got[k].double() - v.double()).square().sum())
        den += float(v.double().square().sum())
        scale = float(v.abs().max())
        if scale > 0:
            e = float((got[k] - v).abs().max()) / scale
            if e > worst[1]:
                worst = (k, e)
    return (num / den) ** 0.5, worst


def wide_tc_chain(spec: O.NerfSpec, w, x, cot, noise, rnd, stats=None):
    """-> gradient dict in state-dict layout.  rnd: fp16 rounding of every tensor-core operand and tape image, or identity.
    The layer engine's arithmetic (fp32 rgb head); the fused engine's images are the same up to fp32 summation order."""
    L, layers, in_xyz = spec.layer_dim, spec.layers, spec.in_xyz
    R = lambda t: rnd(t)                                                              # noqa: E731
    mm = lambda a, b: a @ b                                                           # fp32 accumulation
    # ---- recording forward (layer_launch with a tape)
    pe = R(O.embed(x[:, :spec.xyz_dim], spec.pos_xyz_dim))
    aux = []
    if spec.pos_dir_dim > 0:
        aux.append(O.embed(x[:, -4:-1], spec.pos_dir_dim))
    ids = x[:, -1].long() if spec.appearance_dim > 0 else None
    if spec.appearance_dim > 0:
        aux.append(w['embedding_a.weight'][ids])
    aux = R(torch.cat(aux, -1))
    h, xin = [], []
    cur = pe
    for i in range(layers):
        inp = torch.cat([pe, cur], -1) if i in spec.skip_layers else cur
        xin.append(inp)
        cur = R(torch.relu(mm(inp, R(w[f'xyz_encodings.{i}.0.weight']).t()) + w[f'xyz_encodings.{i}.0.bias']))
        h.append(cur)
    sig_pre = mm(h[-1], w['sigma.weight'].t())[:, 0] + w['sigma.bias'] + noise.view(-1)      # fp32, CUDA cores
    f = R(mm(h[-1], R(w['xyz_encoding_final.weight']).t()) + w['xyz_encoding_final.bias'])
    fx = torch.cat([f, aux], -1)
    g = R(torch.relu(mm(fx, R(w['dir_a_encoding.0.weight']).t()) + w['dir_a_encoding.0.bias']))
    lin = mm(g, w['rgb.weight'].t()) + w['rgb.bias']
    s = torch.sigmoid(lin) if spec.rgb_dim == 3 else lin

    # ---- head stage (tc_layer_head_dgrad_kernel), fp32
    S = grad_scale(cot)
    go_rgb, go_sig = cot[:, :spec.rgb_dim], cot[:, spec.rgb_dim]
    if spec.shifted_softplus:
        y = sig_pre - 1
        dsp = torch.where(y > 20, torch.ones_like(y), 1 / (1 + torch.exp(-y)))
    else:
        dsp = (sig_pre > 0).to(sig_pre.dtype)
    ds = go_sig * dsp
    d = go_rgb * (1 - s) * s if spec.rgb_dim == 3 else go_rgb
    dzg = mm(d, w['rgb.weight']) * (g > 0)                                           # fp32, unscaled
    dzg_img = R(dzg * S)

    G = {k: torch.zeros_like(v) for k, v in w.items()}

    def wop(name, dz_img, xx):                                                        # tc_wgrad_kernel: dZ^T X / S
        G[name + '.weight'] += mm(dz_img.t(), xx) / S
        G[name + '.bias'] += dz_img.sum(0) / S

    # ---- heads (tc_heads_wgrad_kernel) and the embedding (per-image sums x W_e, tc_emb_grad_kernel)
    G['sigma.weight'] += mm(ds.unsqueeze(0), h[-1])
    G['sigma.bias'] += ds.sum().view(1)
    G['rgb.weight'] += mm(d.t(), g)
    G['rgb.bias'] += d.sum(0)
    if spec.appearance_dim > 0:
        sums = torch.zeros(spec.appearance_count, L // 2, dtype=dzg.dtype).index_add_(0, ids, dzg)
        G['embedding_a.weight'] += mm(sums, w['dir_a_encoding.0.weight'][:, L + spec.in_dir:])
    # ---- data-gradient chain (tc_layer_gemm_kernel<false, true>) interleaved with the weight gradients
    Wd = w['dir_a_encoding.0.weight']
    wop('dir_a_encoding.0', dzg_img, fx)
    df = R(mm(dzg_img, R(Wd[:, :L])))                                                 # no mask: F has no activation
    wop('xyz_encoding_final', df, h[-1])
    dz = R((mm(df, R(w['xyz_encoding_final.weight'])) + (ds * S).unsqueeze(-1) * w['sigma.weight']) * (h[-1] > 0))
    if stats is not None:
        stats.append(('S', S))
    for i in range(layers - 1, -1, -1):
        if stats is not None:
            stats.append((f'max |S dZ_{i}|', float(dz.abs().max())))
        wop(f'xyz_encodings.{i}.0', dz, xin[i])
        if i == 0:
            break
        Wi = w[f'xyz_encodings.{i}.0.weight']
        Wh = Wi[:, in_xyz:] if i in spec.skip_layers else Wi                          # hidden columns only
        dz = R(mm(dz, R(Wh)) * (h[i - 1] > 0))
    return G


# ------------------------------------------------------------------------------------------------------------------------
# one stage at a time: each returns (v, beta) in float64, v before the stage's fp16 rounding and post-operation
# ------------------------------------------------------------------------------------------------------------------------
def dot_beta(a, b_t, n, extra=0.0):
    """beta of fp32 sums (a @ b_t) of n products (+ extra, the magnitudes of further fp32 addends)."""
    return C_DOT * (n + 1) * U32 * ((a.abs() @ b_t.abs()) + extra)


def pe_features(x, n_freqs):
    """[x, sin(2^k x), cos(2^k x)]_k in float64 (O.embed's column order) and the encoder's fp32 bound."""
    v = O.embed(x.double(), n_freqs)
    beta = torch.full_like(v, PE_BETA)
    beta[:, :x.shape[1]] = 0.0                   # the inputs themselves are fp32 values
    return v, beta


def pe_band_fp32(x, n_freqs):
    """The fast encoder's recurrence (pe_band, mn_mlp_tc.cu) in fp32, in O.embed's column order."""
    x = x.float()
    parts = [x]
    s = c = None
    for k in range(n_freqs):
        if k % 4 == 0:
            a = x * (2.0 ** k)
            s, c = torch.sin(a), torch.cos(a)
        else:
            s, c = (2.0 * s) * c, 1.0 - (2.0 * s) * s
        parts += [s, c]
    return torch.cat(parts, -1)


def linear_fwd(X, W, b, w16=True):
    """fp16 X (the kernel's input image) times W (fp16-rounded by the pack when w16), fp32 accumulation, + fp32 bias."""
    Wk = h16(W.float()).double() if w16 else W.double()
    v = X @ Wk.t() + b.double()
    return v, dot_beta(X, Wk.t(), X.shape[1], b.double().abs())


def sigma_pre(H16, sw, sb, noise, fused):
    """fp32 sigma pre-activation (with the density noise) from the last trunk image H16."""
    swd = sw.double().view(-1)
    v = H16 @ swd + float(sb) + noise
    beta = dot_beta(H16, swd.view(-1, 1), H16.shape[1], abs(float(sb)) + noise.abs().view(-1, 1)).view(-1)
    if fused:      # summed from the fp32 values before their fp16 rounding
        beta = beta + half_ulp16(H16) @ swd.abs()
    return v, beta


def rgb_head(G16, Wr, br, fused):
    """rgb pre-activation; the fused engine's is an MMA with fp16 weights, the layer engine's fp32 CUDA-core sums."""
    return linear_fwd(G16, Wr, br, w16=fused)


def head_grads(spec, go, bw, tape_rgb, pre):
    """tc_head_grad: (d [n, rgb_dim], dsigma [n]) and their fp32 bounds, from the fp32 head block the forward wrote."""
    R = spec.rgb_dim
    g = go.double() * bw.view(-1, 1)
    if R == 3:
        c = tape_rgb.double()
        d = (g[:, :3] * (1 - c)) * c
        bd = 4 * U32 * d.abs()
    else:
        d = g[:, :R]
        bd = U32 * d.abs()
    pre = pre.double()
    if spec.shifted_softplus:
        y = pre - 1
        dsp = torch.where(y > 20, torch.ones_like(y), 1 / (1 + torch.exp(-y)))
        tol = 8 * U32
    else:
        dsp = (pre > 0).double()
        tol = U32
    ds = g[:, R] * dsp
    return d, bd, ds, tol * ds.abs()


def dz_g(d, Wr, G16):
    """unscaled fp32 dZ_G = mask(G > 0) (W_rgb^T d) (tc_rgb_dgrad8) and its bound."""
    Wd = Wr.double()
    v = (d @ Wd) * (G16 > 0)
    return v, dot_beta(d, Wd, d.shape[1]) * (G16 > 0)


def dgrad(dZ16, W, extra=None):
    """fp16 dZ (an image, S-scaled) times the fp16 transposed weights [out, in_hidden], fp32 accumulation [+ extra, fp32]."""
    Wk = h16(W.float()).double()
    v = dZ16 @ Wk
    e = 0.0 if extra is None else extra.abs()
    if extra is not None:
        v = v + extra
    return v, dot_beta(dZ16, Wk, dZ16.shape[1], e)


def wgrad(dZ16, X16, S):
    """dW = dZ^T X / S and db = sum dZ / S (tc_wgrad_kernel) over the n rows of the sub-module."""
    n = dZ16.shape[0]
    v = dZ16.t() @ X16 / S
    vb = dZ16.sum(0) / S
    ones = torch.ones(n, 1, dtype=dZ16.dtype)
    return v, dot_beta(dZ16.t(), X16, n) / S, vb, dot_beta(dZ16.t(), ones, n).view(-1) / S


def fp32_sum(g, X16):
    """sum_r g[r] X[r] with fp32 g (head gradients): tc_heads_wgrad_kernel."""
    return g.t() @ X16, dot_beta(g.t(), X16, g.shape[0])


# ------------------------------------------------------------------------------------------------------------------------
# criteria
# ------------------------------------------------------------------------------------------------------------------------
class Report:
    """Per stage: elements checked, failures, the largest error / beta ratio beyond fp16 rounding, the share of elements one
    fp16 step off the rounded reference (the interval case)."""

    def __init__(self):
        self.rows = []

    def img(self, name, k, v, beta, op=lambda t: t, slope=1.0):
        k, v, beta = k.double(), v.double(), beta.double()
        lo, hi = h16(op(v - beta)), h16(op(v + beta))
        bad = ~((k >= lo) & (k <= hi))
        ref = h16(op(v))
        off = k != ref
        excess = ((k - op(v)).abs() - half_ulp16(k)).clamp(min=0)
        ratio = excess / (beta * slope).clamp(min=1e-300)
        ratio = torch.where(excess > 0, ratio, torch.zeros_like(ratio))
        self._add(name, k.numel(), bad, ratio, off)

    def f32(self, name, k, v, beta):
        k, v, beta = k.double(), v.double(), beta.double()
        err = (k - v).abs()
        bad = err > beta
        ratio = torch.where(err > 0, err / beta.clamp(min=1e-300), torch.zeros_like(err))
        self._add(name, k.numel(), bad, ratio, err > 0)

    def exact(self, name, k, v):
        bad = k.double() != v.double()
        self._add(name, k.numel(), bad, bad.double(), bad)

    def _add(self, name, n, bad, ratio, off):
        self.rows.append(dict(stage=name, n=int(n), fail=int(bad.sum()), ratio=float(ratio.max()) if n else 0.0,
                              off=float(off.double().mean()) if n else 0.0))

    def failures(self):
        return [r for r in self.rows if r['fail']]

    def text(self):
        return '\n'.join(f"  {r['stage']:<34} n {r['n']:>9}  fail {r['fail']:>6}  max err/beta {r['ratio']:.3f}  "
                         f"one-ulp share {r['off']:.4f}" for r in self.rows)


def mask_op(m, S):
    return lambda t: torch.where(m, t * S, torch.zeros_like(t))


def relu(t):
    return t.clamp(min=0)


# ------------------------------------------------------------------------------------------------------------------------
# the whole check of one sub-module's rows
# ------------------------------------------------------------------------------------------------------------------------
def check_stages(spec: O.NerfSpec, w, cap, fused: bool, rep: Report, tag=''):
    """cap: what the kernels wrote for the slots of one sub-module (float64 unless noted):
      valid [n] bool (the slot holds a row), x [n, cols] the slot's input row, noise [n], go [n, rgb_dim + 1] upstream
      gradient, bw [n] blend weight, xpe [n, kpe], xaux [n, kaux], img[j] [n, cols] for j = trunk layers, F, G,
      sig [n], rgb [n, 3], id [n], S, gf32 [n, 1 + rgb_dim], dz {j: [n, cols]} (dZ images present), emb_sum
      [app_count, emb_k] or None, grads {state-dict key: tensor}, and optional `seed_grads` {key: (v, tol)} for tensors whose
      dZ is not resident (compared at a per-tensor tolerance instead)."""
    check_forward(spec, w, cap, fused, rep, tag)
    check_backward(spec, w, cap, fused, rep, tag)


def app_in_dira(spec: O.NerfSpec) -> bool:
    """The appearance embedding is an input of dir_a_encoding (not the affine colour transform)."""
    return spec.appearance_dim > 0 and not spec.affine_appearance


def head_input(spec: O.NerfSpec, img):
    """The fp16 image the rgb head reads: G, or the last trunk image without dir_a_encoding (nerf.py:154)."""
    L, layers = spec.layer_dim, spec.layers
    return img[layers + 1][:, :L // 2] if spec.has_dir_a else img[layers - 1][:, :L]


def check_forward(spec: O.NerfSpec, w, cap, fused: bool, rep: Report, tag=''):
    """The recording forward of one sub-module's slots: encoder tiles, every activation image from the kernel's previous one, and
    the fp32 head block (sigma pre-activation; the colour / first 3 SH channels unless the rgb goes through the affine transform,
    which only `out` holds: check_output).  cap holds the forward entries of check_stages; without dir_a_encoding img has the
    trunk images only."""
    L, layers, in_xyz, R = spec.layer_dim, spec.layers, spec.in_xyz, spec.rgb_dim
    half = L // 2
    val = cap['valid']
    img = cap['img']
    p = f'{tag}' if tag else ''
    # ---- encoder tiles
    x = cap['x'][val]
    v, b = pe_features(x[:, :spec.xyz_dim], spec.pos_xyz_dim)
    rep.img(p + 'encoder xyz PE', cap['xpe'][val][:, :in_xyz], v, b)
    if cap['xpe'].shape[1] > in_xyz:
        rep.exact(p + 'encoder PE padding', cap['xpe'][:, in_xyz:], torch.zeros_like(cap['xpe'][:, in_xyz:]))
    col = 0
    if spec.pos_dir_dim > 0:
        v, b = pe_features(x[:, -4:-1], spec.pos_dir_dim)
        rep.img(p + 'encoder dir PE', cap['xaux'][val][:, :spec.in_dir], v, b)
        col = spec.in_dir
    ids = x[:, -1].long() if spec.appearance_dim > 0 else None
    n_aux = col
    if app_in_dira(spec):
        e = w['embedding_a.weight'][ids].double()
        rep.img(p + 'encoder embedding', cap['xaux'][val][:, col:col + spec.appearance_dim], e, torch.zeros_like(e))
        n_aux += spec.appearance_dim
    if cap['xaux'].shape[1] > n_aux:
        rep.exact(p + 'encoder aux padding', cap['xaux'][:, n_aux:], torch.zeros_like(cap['xaux'][:, n_aux:]))
    rep.exact(p + 'encoder padding rows', cap['xpe'][~val], torch.zeros_like(cap['xpe'][~val]))

    # ---- forward images, each from the kernel's previous image
    pe16 = cap['xpe'][:, :in_xyz]
    for i in range(layers):
        prev = pe16 if i == 0 else img[i - 1][:, :L]
        X = torch.cat([pe16, prev], -1) if (i in spec.skip_layers and i > 0) else prev
        v, b = linear_fwd(X, w[f'xyz_encodings.{i}.0.weight'], w[f'xyz_encodings.{i}.0.bias'])
        rep.img(p + f'fwd H{i}', img[i][:, :L], v, b, relu)
    H = img[layers - 1][:, :L]
    if spec.has_dir_a:
        v, b = linear_fwd(H, w['xyz_encoding_final.weight'], w['xyz_encoding_final.bias'])
        rep.img(p + 'fwd F', img[layers][:, :L], v, b)
        aux16 = cap['xaux'][:, :n_aux]
        FX = torch.cat([img[layers][:, :L], aux16], -1)
        v, b = linear_fwd(FX, w['dir_a_encoding.0.weight'], w['dir_a_encoding.0.bias'])
        rep.img(p + 'fwd G', img[layers + 1][:, :half], v, b, relu)
    for j in range(len(img)):                      # the layer engine's padding columns hold exactly 0
        if img[j].shape[1] > (half if j == layers + 1 else L):
            pad = img[j][:, half if j == layers + 1 else L:]
            rep.exact(p + f'fwd image {j} padding', pad, torch.zeros_like(pad))
    noise = cap['noise'].double()
    v, b = sigma_pre(H[val], w['sigma.weight'], w['sigma.bias'], noise[val], fused)
    rep.f32(p + 'head sigma pre-activation', cap['sig'][val], v, b)
    if not spec.affine_appearance:
        v, b = rgb_head(head_input(spec, img)[val], w['rgb.weight'], w['rgb.bias'], fused)
        if R == 3:
            c = torch.sigmoid(v)
            rep.f32(p + 'head rgb', cap['rgb'][val], c, 0.25 * b + 4 * U32)
        else:
            rep.f32(p + 'head rgb', cap['rgb'][val], v[:, :3], b[:, :3])
    if ids is not None:
        rep.exact(p + 'head image id', cap['id'][val], x[:, -1].double())


def check_backward(spec: O.NerfSpec, w, cap, fused: bool, rep: Report, tag=''):
    """The backward of one sub-module's slots (check_stages), seeded from the kernels' forward tape and head-gradient blocks."""
    L, layers, in_xyz, R = spec.layer_dim, spec.layers, spec.in_xyz, spec.rgb_dim
    half = L // 2
    val = cap['valid']
    S = cap['S']
    img = cap['img']
    p = f'{tag}' if tag else ''
    x = cap['x'][val]
    ids = x[:, -1].long() if spec.appearance_dim > 0 else None
    H = img[layers - 1][:, :L]
    G16 = img[layers + 1][:, :half]
    aux16 = cap['xaux'][:, :spec.in_dir + spec.appearance_dim]
    FX = torch.cat([img[layers][:, :L], aux16], -1)
    pe16 = cap['xpe'][:, :in_xyz]
    xin = [torch.cat([pe16, img[i - 1][:, :L]], -1) if (i in spec.skip_layers and i > 0) else (pe16 if i == 0 else img[i - 1][:, :L])
           for i in range(layers)]

    # ---- backward head stage
    d, bd, ds, bds = head_grads(spec, cap['go'], cap['bw'], cap['rgb'], cap['sig'])
    gf = cap['gf32']
    rep.f32(p + 'head grad dsigma', gf[:, 0], ds, bds)
    rep.f32(p + 'head grad d rgb', gf[:, 1:1 + R], d, bd)
    dkern, dskern = gf[:, 1:1 + R], gf[:, 0]                 # seeds of the later stages
    vzg, bzg = dz_g(dkern, w['rgb.weight'], G16)
    dz = cap['dz']
    gmask = G16 > 0
    if layers + 1 in dz:
        rep.img(p + 'dZ_G', dz[layers + 1][:, :half], vzg, bzg, mask_op(gmask, S), S)
    # ---- data-gradient chain, each dZ image from the kernel's previous one (those still resident)
    Wd = w['dir_a_encoding.0.weight']
    if layers + 1 in dz and layers in dz:
        v, b = dgrad(dz[layers + 1][:, :half], Wd[:, :L])
        rep.img(p + 'dZ_F', dz[layers][:, :L], v, b, lambda t: t)
    if layers in dz and layers - 1 in dz:
        extra = (dskern * S).view(-1, 1) * w['sigma.weight'].double().view(1, -1)
        v, b = dgrad(dz[layers][:, :L], w['xyz_encoding_final.weight'], extra)
        m = H > 0
        rep.img(p + f'dZ_{layers - 1}', dz[layers - 1][:, :L], v, b, mask_op(m, 1.0), 1.0)
        rep.exact(p + f'dZ_{layers - 1} zero where masked', dz[layers - 1][:, :L][~m], torch.zeros(int((~m).sum()), dtype=torch.float64))
    for i in range(layers - 1, 0, -1):
        if i in dz and i - 1 in dz:
            Wi = w[f'xyz_encodings.{i}.0.weight']
            Wh = Wi[:, in_xyz:] if i in spec.skip_layers else Wi
            v, b = dgrad(dz[i][:, :L], Wh)
            m = img[i - 1][:, :L] > 0
            rep.img(p + f'dZ_{i - 1}', dz[i - 1][:, :L], v, b, mask_op(m, 1.0), 1.0)
            rep.exact(p + f'dZ_{i - 1} zero where masked', dz[i - 1][:, :L][~m], torch.zeros(int((~m).sum()), dtype=torch.float64))
    for j, z in dz.items():
        rep.f32(p + f'dZ image {j} below fp16 max', z.abs().max().view(1), torch.zeros(1, dtype=torch.float64),
                torch.full((1,), 65504.0 / 2, dtype=torch.float64))

    # ---- parameter gradients, per element, from the kernel's own images
    grads = cap['grads']

    def wchk(name, Z, X):
        v, b, vb, bb = wgrad(Z, X, S)
        rep.f32(p + f'grad {name}.weight', grads[name + '.weight'], v, b)
        rep.f32(p + f'grad {name}.bias', grads[name + '.bias'], vb, bb)

    if layers + 1 in dz:
        wchk('dir_a_encoding.0', dz[layers + 1][:, :half], FX)
    if layers in dz:
        wchk('xyz_encoding_final', dz[layers][:, :L], H)
    for i in range(layers):
        if i in dz:
            wchk(f'xyz_encodings.{i}.0', dz[i][:, :L], xin[i])
    for k, (v, tol) in cap.get('seed_grads', {}).items():
        scale = float(v.abs().max())
        rep.f32(p + f'grad {k} (restatement)', grads[k], v, torch.full_like(v, tol * max(scale, 1e-30)))
    v, b = fp32_sum(dskern.view(-1, 1), H)
    rep.f32(p + 'grad sigma.weight', grads['sigma.weight'], v, b)
    v, b = fp32_sum(dskern.view(-1, 1), torch.ones(H.shape[0], 1, dtype=torch.float64))
    rep.f32(p + 'grad sigma.bias', grads['sigma.bias'], v.view(-1), b.view(-1))
    v, b = fp32_sum(dkern, G16)
    rep.f32(p + 'grad rgb.weight', grads['rgb.weight'], v, b)
    v, b = fp32_sum(dkern, torch.ones(H.shape[0], 1, dtype=torch.float64))
    rep.f32(p + 'grad rgb.bias', grads['rgb.bias'], v.view(-1), b.view(-1))
    if ids is not None and cap.get('emb_sum') is not None:
        idv = cap['id'].long().clamp(0, spec.appearance_count - 1)
        vv, bb = vzg * val.view(-1, 1), bzg * val.view(-1, 1)
        sums = torch.zeros(spec.appearance_count, half, dtype=torch.float64).index_add_(0, idv, vv)
        sb = torch.zeros_like(sums).index_add_(0, idv, bb) + C_DOT * H.shape[0] * U32 * \
            torch.zeros_like(sums).index_add_(0, idv, vv.abs())
        es = cap['emb_sum'][:, :half]
        rep.f32(p + 'embedding per-image sums', es, sums, sb)
        We = Wd[:, L + spec.in_dir:].double()
        v = es @ We
        b = dot_beta(es, We, half)
        rep.f32(p + 'grad embedding_a.weight', grads['embedding_a.weight'], v, b)
        unused = torch.ones(spec.appearance_count, dtype=torch.bool)
        unused[idv[val]] = False
        rep.exact(p + 'grad embedding_a.weight unused ids', grads['embedding_a.weight'][unused],
                  torch.zeros_like(grads['embedding_a.weight'][unused]))


# ------------------------------------------------------------------------------------------------------------------------
# output assembly: what a call writes to `out` (tc_emit_rgb and the sigma epilogue of either engine, then combine_kernel)
# ------------------------------------------------------------------------------------------------------------------------
def sigma_act(spec: O.NerfSpec, pre):
    """sigma_activation of the kernel's fp32 pre-activation, (v, beta).  ReLU (fmaxf) is exact.  mn_softplus_shifted rounds
    y = pre - 1 (U32 |y|), then log1pf(expf(y)): expf within 2 ulps (4 U32 of e^y, which moves softplus by 4 U32 sigmoid(y))
    and log1pf within 1 ulp (2 U32 softplus(y)); beta is twice their sum.  Above y = 20 it returns y, 2e-9 from softplus(y)."""
    pre = pre.double()
    if not spec.shifted_softplus:
        return pre.clamp(min=0), torch.zeros_like(pre)
    y = pre - 1
    v = torch.logaddexp(y, torch.zeros_like(y))
    sg = torch.sigmoid(y)
    return v, 2 * (sg * (U32 * y.abs() + 4 * U32) + 2 * U32 * v)


def rgb_out(spec: O.NerfSpec, w, src16, ids, fused: bool):
    """The rgb columns of one slot's output from the head's input image, (v [n, rgb_dim], beta): the rgb Linear (rgb_head), then
    tc_emit_rgb - the affine transform T = affine(embedding_a[id]) (fp32 fmaf chains over the embedding), y_c = sum_k T[c][k]
    r_k + T[c][3] (three roundings), and the sigmoid of a colour head (1 / (1 + expf(-y)): 2 ulps of expf, one add and one
    divide, 8 U32 of the value; the slope of the sigmoid is at most 1/4)."""
    v, b = rgb_head(src16, w['rgb.weight'], w['rgb.bias'], fused)
    if spec.affine_appearance and spec.appearance_dim > 0:
        e = w['embedding_a.weight'].double()[ids]
        A, ab = w['affine.weight'].double(), w['affine.bias'].double()
        T = (e @ A.t() + ab).view(-1, 3, 4)
        bT = dot_beta(e, A.t(), e.shape[1], ab.abs()).view(-1, 3, 4)
        prod = T[:, :, :3] * v.unsqueeze(1)
        y = prod.sum(-1) + T[:, :, 3]
        by = ((T[:, :, :3].abs() + bT[:, :, :3]) * b.unsqueeze(1) + v.abs().unsqueeze(1) * bT[:, :, :3]).sum(-1) + bT[:, :, 3] \
            + 4 * U32 * (prod.abs().sum(-1) + T[:, :, 3].abs())
        v, b = y, by
    if spec.rgb_dim == 3:
        c = torch.sigmoid(v)
        return c, 0.25 * b + 8 * U32 * c
    return v, b


def slot_outputs(spec: O.NerfSpec, w, cap, fused: bool):
    """Per valid slot of one sub-module, before the blend weight: v / beta [n, rgb_dim + 1] restated from the kernel's head input
    image and fp32 sigma pre-activation, and `exact` the colour (or first 3 SH channels) of the fp32 head block, which the
    kernel stores to `out` unchanged (None for the affine head, which the head block does not hold)."""
    val = cap['valid']
    ids = cap['x'][val][:, -1].long() if spec.appearance_dim > 0 else None
    vr, br = rgb_out(spec, w, head_input(spec, cap['img'])[val], ids, fused)
    vs, bs = sigma_act(spec, cap['sig'][val])
    exact = None if spec.affine_appearance else cap['rgb'][val][:, :min(spec.rgb_dim, 3)]
    return dict(v=torch.cat([vr, vs.view(-1, 1)], 1), beta=torch.cat([br, bs.view(-1, 1)], 1), exact=exact)


def check_output(spec: O.NerfSpec, out, pieces, rep: Report, tag=''):
    """out [n, rgb_dim + 1]: the call's output for n rows.  pieces: per sub-module in ascending order, (rows [k] indices into out,
    bw [k] fp32 blend weights or None, slot_outputs of those slots).  A blended call stores x * w per slot (one fp32 rounding)
    and combine_kernel sums a row's slots from 0 in ascending sub-module order; an unblended one stores x.  The head block's
    colour then gives `out` bit for bit (float32 arithmetic here in the kernel's order); every column is within the sum of the
    slots' betas, their products' and the sum's roundings (k U32 sum |x w| for k slots) of the float64 restatement."""
    p = f'{tag}' if tag else ''
    n, C = out.shape
    m = min(spec.rgb_dim, 3)
    v = torch.zeros(n, C, dtype=torch.float64)
    b = torch.zeros_like(v)
    mag = torch.zeros_like(v)
    cnt = torch.zeros(n, 1, dtype=torch.float64)
    acc = torch.zeros(n, m, dtype=torch.float32)
    exact = all(so['exact'] is not None for _, _, so in pieces)
    for rows, bw, so in pieces:
        wv = torch.ones(len(rows), 1, dtype=torch.float64) if bw is None else bw.double().view(-1, 1)
        val = so['v'] * wv
        v.index_add_(0, rows, val)
        b.index_add_(0, rows, so['beta'] * wv + (0.0 if bw is None else U32 * val.abs()))
        mag.index_add_(0, rows, val.abs())
        cnt.index_add_(0, rows, torch.ones(len(rows), 1, dtype=torch.float64))
        if exact:
            x32 = so['exact'].float()
            acc[rows] = acc[rows] + (x32 if bw is None else x32 * bw.float().view(-1, 1))
    b = b + cnt * U32 * mag
    out = out.double()
    rep.f32(p + 'out rgb', out[:, :C - 1], v[:, :C - 1], b[:, :C - 1])
    rep.f32(p + 'out sigma', out[:, C - 1], v[:, C - 1], b[:, C - 1])
    if exact:
        rep.exact(p + 'out rgb = head block (bitwise)', out[:, :m], acc.double())


def seeded_chain(spec: O.NerfSpec, w, cap, S):
    """The layer engine's dZ chain below the resident images, restated with fp16 rounding and seeded with the kernel's forward
    tape (masks, X) and head-gradient blocks: {state-dict key: value} of the weight / bias gradients it yields."""
    L, layers, in_xyz = spec.layer_dim, spec.layers, spec.in_xyz
    half = L // 2
    img = cap['img']
    H = img[layers - 1][:, :L]
    dzg = cap['dz'][layers + 1][:, :half]
    out = {}
    pe16 = cap['xpe'][:, :in_xyz]

    def X(i):
        prev = pe16 if i == 0 else img[i - 1][:, :L]
        return torch.cat([pe16, prev], -1) if (i in spec.skip_layers and i > 0) else prev

    def put(name, Z, XX):
        out[name + '.weight'] = Z.t() @ XX / S
        out[name + '.bias'] = Z.sum(0) / S

    df = h16(dgrad(dzg, w['dir_a_encoding.0.weight'][:, :L])[0])
    put('xyz_encoding_final', df, H)
    extra = (cap['gf32'][:, 0] * S).view(-1, 1) * w['sigma.weight'].double().view(1, -1)
    dz = h16(dgrad(df, w['xyz_encoding_final.weight'], extra)[0] * (H > 0))
    for i in range(layers - 1, -1, -1):
        put(f'xyz_encodings.{i}.0', dz, X(i))
        if i == 0:
            break
        Wi = w[f'xyz_encodings.{i}.0.weight']
        dz = h16(dgrad(dz, Wi[:, in_xyz:] if i in spec.skip_layers else Wi)[0] * (img[i - 1][:, :L] > 0))
    return out
