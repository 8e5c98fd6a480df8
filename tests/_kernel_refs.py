"""float64 restatements of the row-wise and fp32 attention entry points of include/mer_b200.h, of the fusion nets'
dropout hash, loss, gradients and Adam, and the small helpers the kernel-level GPU tests share (environment switches,
guarded output buffers).  Every function takes torch tensors on any device and computes in float64 on that device;
tests/test_kernel_refs.py checks them on the CPU against torch's own operators."""
import contextlib
import math
import os

import numpy as np
import torch
import torch.nn.functional as F

U32 = 2.0 ** -24  # unit roundoff of fp32 (round to nearest)


@contextlib.contextmanager
def env(name, value):
    """Set (value is a string) or unset (None) an environment variable and restore it afterwards."""
    old = os.environ.get(name)
    try:
        if value is None:
            os.environ.pop(name, None)
        else:
            os.environ[name] = str(value)
        yield
    finally:
        if old is None:
            os.environ.pop(name, None)
        else:
            os.environ[name] = old


def guarded(rows, cols, dtype, device, guard=2, fill=float("nan")):
    """A [rows, cols] view between `guard` rows that must keep `fill`: returns (whole buffer, view)."""
    buf = torch.full((rows + 2 * guard, cols), fill, dtype=dtype, device=device)
    return buf, buf[guard:guard + rows]


def guards_intact(buf, rows, guard=2):
    g = torch.cat([buf[:guard], buf[guard + rows:]])
    return bool(torch.isnan(g).all())


def bits(x):
    """Bit pattern of an fp32 / fp16 tensor (so that -0.0 != 0.0 and NaN == NaN in comparisons)."""
    return x.contiguous().view(torch.int32 if x.dtype == torch.float32 else torch.int16)


def round_tf32_ties_away(x):
    """cvt.rna.tf32.f32 on fp32 values: round to 10 explicit mantissa bits, ties away from zero."""
    b = x.contiguous().view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32)


def round_bf16_nearest_even(x):
    b = x.contiguous().view(torch.int32)
    return ((b + 0x7FFF + ((b >> 16) & 1)) & ~0xFFFF).view(torch.float32)


def split_halves(xs):
    """(hi, lo) of split bf16 rows (128-byte groups of 32 bf16 hi | 32 bf16 lo held in an fp32-typed tensor)."""
    K = xs.shape[-1]
    b = xs.contiguous().view(torch.bfloat16).view(*xs.shape[:-1], K // 32, 2, 32).float()
    return b[..., 0, :].reshape(*xs.shape[:-1], K), b[..., 1, :].reshape(*xs.shape[:-1], K)


def layernorm(x, gamma, beta, eps):
    """torch.nn.LayerNorm: biased variance about the mean, eps inside the square root."""
    x = x.double()
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + eps) * gamma.double() + beta.double()


def layernorm_bound(x, gamma, y_ref, eps):
    """Elementwise bound of a two-pass fp32 LayerNorm against float64.  The fp32 row sum (a lane's sequential partial
    sum, then five shuffle steps) leaves the mean off by a few u * max|x|; that shifts every centred value, i.e. moves y
    by |gamma| * dmean / sigma.  Centring, the squares' sum, 1 / sqrt and the affine add a few u relative to each of
    |gamma (x - mean) / sigma| and |y|.  8 u for each term; u = 2^-24."""
    x = x.double()
    mu = x.mean(-1, keepdim=True)
    sig = torch.sqrt(((x - mu) ** 2).mean(-1, keepdim=True) + eps)
    g = gamma.double().abs()
    return 8 * U32 * (g * (x.abs().amax(-1, keepdim=True) + (x - mu).abs()) / sig + y_ref.abs()) + 1e-30


def gelu_erf(x):
    x = x.double()
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def segment_reduce(x, begins, ends, mean):
    x = x.double()
    out = torch.zeros(len(begins), x.shape[1], dtype=torch.float64, device=x.device)
    for s, (a, b) in enumerate(zip(begins, ends)):
        if b > a:
            out[s] = x[a:b].mean(0) if mean else x[a:b].sum(0)
    return out


def wave_normalize(x):
    """HF Wav2Vec2FeatureExtractor.zero_mean_unit_var_norm: (x - mean) / sqrt(var + 1e-7), biased variance."""
    x = x.double()
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) / torch.sqrt(var + 1e-7)


# ---- HuBERT front end: conv0 (mer_hubert_conv0) ------------------------------------------------------------------------
# Elementwise bounds of the kernels against the float64 reference on the same fp32 samples, u = 2^-24, A = |w| * |x|
# (the conv of the absolute values; + |bias| for the LayerNorm form), n = the clip's frame count.
#
# GroupNorm form (conv0_moments / conv0_coef / conv0_apply(2)):
#   conv     the fp32 chain of 10 fma: <= 10 u A (every rounding is <= u times a partial sum, and |partial| <= A).
#   mean     rounded to float: u |mean|; its double sums add <= (n + 11) 2^-53 mean_t(A).
#   variance q / n - mean^2 from double moments: each moment is a sum of n exact products (in chunks, in any order),
#            and q combines the 55 products with 55 more fma, so |dvar| <= (3 n + 100) 2^-53 mean_t(A^2).  Relative to
#            var + eps this is the conditioning kappa = mean_t(A^2) / (var + eps) times (3 n + 100) 2^-53: a clip with a
#            DC offset has a large kappa (the cancellation the double moments exist to absorb).
#   scale    g = gamma * float(1 / sqrt(var + eps)): relative 0.5 |dvar| / (var + eps) + 2 u (the float conversion and
#            the fp32 product with gamma).
#   affine   d = y - mean rounds (u |d|), z = d g + beta rounds once or twice (u (|z| + |d g|)); d carries the conv and
#            mean errors, g its relative error: |dz| <= |g| (10 u A + u |mean| + u |d|) + |d g| rg + u (|z| + |d g|).
#   GELU     slope <= 1.13; gelu_erf_fast's own error <= min(4.7e-7, 2.9e-7 |z|) (mer_common.cuh), + u |GELU|.
#   output   split bf16 hi + lo: 2^-17 relative; fp16: half an ulp, max(2^-11 |v|, 2^-25).
# Second-order terms (a u-sized error of a u-sized error) are covered by the +1 in 11 u for the conv chain.
#
# LayerNorm form (conv0_ln_kernel): the conv + bias chain (11 fma, <= 11 u A) carried through the LayerNorm's
# derivative, |gamma| / sigma (|e| + mean_c |e| + |zhat| mean_c(|zhat| |e|)), plus the two-pass fp32 LayerNorm's own
# error (layernorm_bound), then GELU and the output rounding as above.
#
# What the bounds tell apart (tests/test_kernel_refs.py): a variance divided by n - 1 instead of n (relative 1 / n:
# 6e-5 on a 5 s clip) and an eps of 1e-7 instead of 1e-5 on channels whose variance is not far above eps.
CONV0_EPS = 1e-5
GELU_SLOPE = 1.13
U53 = 2.0 ** -53


def gelu_fast_error(z):
    return torch.minimum(torch.full_like(z, 4.7e-7), 2.9e-7 * z.abs())


def out_rounding(v, f16):
    return torch.clamp(2.0 ** -11 * v.abs(), min=2.0 ** -25) if f16 else 2.0 ** -17 * v.abs()


def speech_like(n, seed, dc=0.0, noise=1.0):
    """A seeded fp32 [n] waveform: a few amplitude-modulated harmonics plus white noise, then `dc` added."""
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(n, dtype=torch.float64) / 16000.0
    f0 = 110.0 + 60.0 * float(torch.rand(1, generator=g))
    x = sum(torch.sin(2 * math.pi * f0 * h * t + float(torch.rand(1, generator=g)) * 6.0) / h for h in (1, 2, 3, 5))
    x = x * (0.6 + 0.4 * torch.sin(2 * math.pi * 3.0 * t))
    return (x + noise * 0.3 * torch.randn(n, generator=g, dtype=torch.float64) + dc).float()


def conv0_weights(seed):
    """(w0 [512, 10], gamma, beta, bias) for conv0 tests: He-scaled taps, with every third channel scaled by 1e-3 and
    every third by 3e-3, so that a normalised clip gives channel variances around eps (1e-5) as well as around 2."""
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(512, 10, generator=g) * math.sqrt(2.0 / 10)
    w[1::3] *= 1e-3
    w[2::3] *= 3e-3
    gamma = 1.0 + 0.1 * torch.randn(512, generator=g)
    beta = 0.1 * torch.randn(512, generator=g)
    bias = 0.05 * torch.randn(512, generator=g)
    return w, gamma, beta, bias


def conv0(wave, w0, bias=None):
    """Conv1d(1 -> 512, k 10, s 5) in float64: (y, A) as [B, T0, 512], A = |w| * |x| (+ |bias|)."""
    x = wave.double()[:, None]
    w = w0.double().reshape(512, 1, 10)
    y = F.conv1d(x, w, None if bias is None else bias.double(), stride=5).transpose(1, 2)
    a = F.conv1d(x.abs(), w.abs(), None if bias is None else bias.double().abs(), stride=5).transpose(1, 2)
    return y, a


def conv0_moments(wave, n):
    """The 10 tap sums X_k = sum_t x[5 t + k] and the 10 x 10 tap products R_kk' of the first n frames of each row."""
    x = wave.double()
    taps = torch.stack([x[:, k:k + 5 * (n - 1) + 1:5] for k in range(10)], -1)   # [B, n, 10]
    return taps.sum(1), taps.transpose(1, 2) @ taps


def conv0_stats_from_moments(X, R, w0, n):
    """Per-channel (mean, biased variance) of conv0 from the moments: sum_k w_k X_k / n and w R w^T / n - mean^2."""
    w = w0.double().reshape(512, 10)
    mean = X @ w.T / n
    q = torch.einsum("ck,bkl,cl->bc", w, R, w)
    return mean, q / n - mean * mean


def hubert_conv0(wave, w0, gamma, beta, family="group", bias=None, frames=None, f16=False, eps=CONV0_EPS,
                 var_div=None):
    """First layer of the feature encoder in float64: conv0, then GroupNorm(512 groups, biased variance over the clip's
    first frames[b] frames, or all) -- family "group" -- or conv bias + LayerNorm(512) -- family "layer" -- then exact
    GELU.  Returns (out [B, T0, 512], elementwise bound of the kernel's error, see above; f16: fp16 output rows).
    var_div (tests of the bound only): divide the sum of squares by frames + var_div instead of frames."""
    y, A = conv0(wave, w0, bias if family == "layer" else None)
    B, T0, _ = y.shape
    g = gamma.double()
    if family == "layer":
        mu = y.mean(-1, keepdim=True)
        sig = torch.sqrt(((y - mu) ** 2).mean(-1, keepdim=True) + eps)
        zh = (y - mu) / sig
        z = zh * g + beta.double()
        e = 11 * U32 * A
        dz = g.abs() / sig * (e + e.mean(-1, keepdim=True) + zh.abs() * (zh.abs() * e).mean(-1, keepdim=True))
        dz = dz + layernorm_bound(y, gamma, z, eps)
    else:
        ns = [T0] * B if frames is None else [int(f) for f in frames]
        mean = torch.stack([y[b, :ns[b]].mean(0) for b in range(B)])[:, None]            # [B, 1, 512]
        ss = torch.stack([((y[b, :ns[b]] - mean[b]) ** 2).sum(0) for b in range(B)])[:, None]
        n = torch.tensor(ns, dtype=torch.float64, device=y.device)[:, None, None]
        var = ss / (n + (var_div or 0))
        A2 = torch.stack([(A[b, :ns[b]] ** 2).mean(0) for b in range(B)])[:, None]
        A1 = torch.stack([A[b, :ns[b]].mean(0) for b in range(B)])[:, None]
        rg = 0.5 * (3 * n + 100) * U53 * A2 / (var + eps) + 2 * U32
        gs = g / torch.sqrt(var + eps)
        d = y - mean
        z = d * gs + beta.double()
        dg = (d * gs).abs()
        dz = gs.abs() * (11 * U32 * A + U32 * mean.abs() + (n + 11) * U53 * A1 + U32 * d.abs()) + dg * rg + \
            U32 * (z.abs() + dg)
    out = gelu_erf(z)
    bound = GELU_SLOPE * dz + gelu_fast_error(z) + U32 * out.abs()
    return out, bound + out_rounding(out, f16 and family != "layer")


# ---- HuBERT front end: hidden_states[0] (mer_hubert_frontend) ----------------------------------------------------------
# The reference is oracle.encoders.hubert_hidden_states(layers=0) in float64, restated stage by stage so that each stage
# can carry an elementwise error bound e next to its value v:
#   linear / conv  v = W a (+ b).  Every error here is treated as the sum of independent, mean-zero roundings (the
#                  probabilistic analysis of Higham and Mary, with lambda = 4 standard deviations): the error carried in,
#                  sqrt(W^2 e^2), plus the stage's own, 4 sqrt(u_op^2 + K u^2) sqrt(W^2 a^2): u_op = the operands'
#                  unit (split bf16 hi + lo for activations and weights, the dropped lo * lo: 2^-15; fp16 or tf32
#                  activations of fp16-exact weights: 2^-11; fp16 rows already rounded: 0), K u the fp32 accumulation
#                  of K products.  The worst case, |W| e and (u_op + K u) |W| |a|, grows by ~sqrt(K) per stage (~40 for
#                  K = 1536, 40^6 over the conv stack) and would bound nothing.
#   GELU           |GELU'(z)| e + 0.4 e^2 (|GELU''| <= 0.8), + gelu_erf_fast's own error and u |v|.
#   LayerNorm      the derivative's gain |gamma| / sigma times e (the rest of the derivative is an orthogonal projection,
#                  which does not enlarge independent errors), + layernorm_bound.
#   rows           + 2^-17 |v| for split-bf16 rows, max(2^-11 |v|, 2^-25) for fp16 rows, u |v| for an fp32 add.
# Unlike the conv0 bound this one is not a worst case; it is far above the errors the front end makes and far below
# the error of a misplaced frame or channel.
LAMBDA = 4.0


def _lin_err(conv, v, e, w, u_op, K):
    return torch.sqrt(conv(e * e, w * w).clamp(min=0.0)) + \
        LAMBDA * math.sqrt(u_op ** 2 + K * U32 ** 2) * torch.sqrt(conv(v * v, w * w).clamp(min=0.0))


def _ln_err(x, e, gamma, beta, eps):
    mu = x.mean(-1, keepdim=True)
    sig = torch.sqrt(((x - mu) ** 2).mean(-1, keepdim=True) + eps)
    zh = (x - mu) / sig
    y = zh * gamma + beta
    return y, gamma.abs() / sig * e + layernorm_bound(x, gamma, y, eps)


def _gelu_err(z, e):
    g = gelu_erf(z)
    slope = (0.5 * (1.0 + torch.erf(z / math.sqrt(2.0))) + z * torch.exp(-0.5 * z * z) / math.sqrt(2 * math.pi)).abs()
    return g, slope * e + 0.4 * e * e + gelu_fast_error(z) + U32 * g.abs()


def fp16_exact_front_end(sd):
    """A copy of a HuBERT-family state dict whose fp16-operand weights are fp16-exact: the positional conv stored as its
    folded `weight` (no weight norm) rounded to fp16, conv1 and conv2, and the data2vec chain's convs."""
    from mertools_b200.encoders import fold_pos_conv_weight
    r16 = lambda v: np.asarray(v, np.float32).astype(np.float16).astype(np.float32)  # noqa: E731
    out = dict(sd)
    pre = "encoder.pos_conv_embed.conv."
    if pre + "parametrizations.weight.original0" in sd:
        out[pre + "weight"] = r16(fold_pos_conv_weight(sd))
        del out[pre + "parametrizations.weight.original0"], out[pre + "parametrizations.weight.original1"]
    for k in list(out):
        if k.startswith(("feature_extractor.conv_layers.1.conv.weight", "feature_extractor.conv_layers.2.conv.weight",
                         "encoder.pos_conv_embed.layers.")) and k.endswith("conv.weight"):
            out[k] = r16(out[k])
    return out


def hubert_hidden0(sd, wave, conv_f16=False, ln_eps=1e-5):
    """(hidden_states[0] [B, T, D], bound) of the HuBERT-family front end on fp32 input values `wave` [B, n] (already
    normalised when the model normalises).  conv_f16: conv1 and conv2 on fp16 operands (group-norm feature encoder).
    The positional conv's unit is 2^-11 in both of its forms (fp16 activations in the windowed GEMM, tf32 in the
    mma.sync kernel).  The fp16-operand weights must be fp16-exact (fp16_exact_front_end): the bound has no term for
    their rounding."""
    dev = wave.device
    t = lambda k: torch.as_tensor(np.asarray(sd[k])).to(dev, torch.float64)  # noqa: E731
    cl = "feature_extractor.conv_layers."
    ln_convs = cl + "1.layer_norm.weight" in sd
    data2vec = "encoder.pos_conv_embed.layers.0.conv.weight" in sd
    stable = ln_convs and not data2vec
    w0 = t(cl + "0.conv.weight").reshape(512, 10)
    b0 = t(cl + "0.conv.bias") if cl + "0.conv.bias" in sd else None
    a, e = hubert_conv0(wave, w0, t(cl + "0.layer_norm.weight"), t(cl + "0.layer_norm.bias"),
                        family="layer" if ln_convs else "group", bias=b0, f16=conv_f16)
    a, e = a.transpose(1, 2), e.transpose(1, 2)                                  # [B, 512, T]
    for i in range(1, 7):
        w = t(cl + f"{i}.conv.weight")
        bias = t(cl + f"{i}.conv.bias") if cl + f"{i}.conv.bias" in sd else None
        conv = lambda x, ww: F.conv1d(x, ww, stride=2)  # noqa: E731
        f16_in = conv_f16 and i <= 2
        z = F.conv1d(a, w, bias, stride=2)
        ez = _lin_err(conv, a, e, w, 0.0 if f16_in else 2.0 ** -15, w.shape[1] * w.shape[2])
        if bias is not None:
            ez = ez + U32 * bias.abs()[:, None]
        if ln_convs:
            z, ez = (v.transpose(1, 2) for v in _ln_err(z.transpose(1, 2), ez.transpose(1, 2),
                                                        t(cl + f"{i}.layer_norm.weight"),
                                                        t(cl + f"{i}.layer_norm.bias"), 1e-5))
        a, e = _gelu_err(z, ez)
        if i < 6:
            e = e + out_rounding(a, conv_f16 and i == 1)
    a, e = _ln_err(a.transpose(1, 2), e.transpose(1, 2), t("feature_projection.layer_norm.weight"),
                   t("feature_projection.layer_norm.bias"), ln_eps)
    e = e + out_rounding(a, False)
    w = t("feature_projection.projection.weight")
    x0 = a @ w.T + t("feature_projection.projection.bias")
    e0 = _lin_err(lambda x, ww: x @ ww.T, a, e, w, 2.0 ** -15, w.shape[1]) + U32 * x0.abs()
    D = x0.shape[-1]
    g = 16
    if data2vec:
        p, ep, l = x0.transpose(1, 2), e0.transpose(1, 2), 0
        while f"encoder.pos_conv_embed.layers.{l}.conv.weight" in sd:
            w = t(f"encoder.pos_conv_embed.layers.{l}.conv.weight")
            k = w.shape[-1]
            conv = lambda x, ww: F.conv1d(x, ww, padding=k // 2, groups=g)  # noqa: E731
            z = F.conv1d(p, w, t(f"encoder.pos_conv_embed.layers.{l}.conv.bias"), padding=k // 2, groups=g)
            ez = _lin_err(conv, p, ep, w, 2.0 ** -11, w.shape[1] * k) + U32 * z.abs()
            ones = torch.ones(D, dtype=torch.float64, device=dev)
            z, ez = _ln_err(z.transpose(1, 2), ez.transpose(1, 2), ones, ones * 0, 1e-5)
            p, ep = (v.transpose(1, 2) for v in _gelu_err(z, ez))
            l += 1
        x = x0 + p.transpose(1, 2)
        ex = e0 + ep.transpose(1, 2) + U32 * x.abs()
    else:
        from oracle.encoders import hubert_pos_conv_weight
        w = hubert_pos_conv_weight(sd, torch.float64).to(dev)
        conv = lambda x, ww: F.conv1d(x, ww, padding=64, groups=g)[:, :, :-1]  # noqa: E731
        xt, et = x0.transpose(1, 2), e0.transpose(1, 2)
        z = conv(xt, w) + t("encoder.pos_conv_embed.conv.bias")[:, None]
        ez = _lin_err(conv, xt, et, w, 2.0 ** -11, w.shape[1] * 128) + U32 * z.abs()
        p, ep = _gelu_err(z, ez)
        x = x0 + p.transpose(1, 2)
        ex = e0 + ep.transpose(1, 2) + U32 * x.abs()
    if not stable:
        x, ex = _ln_err(x, ex, t("encoder.layer_norm.weight"), t("encoder.layer_norm.bias"), ln_eps)
    return x, ex


def attention_packed(qkv, cu, heads):
    """softmax(Q K^T / 8) V per (sequence, head) of packed [tokens, 3 * heads * 64] rows.  Returns (ctx, P |V|, A): P |V|
    is the scale of the error a perturbed probability leaves, A [tokens, heads * 64] the row's max_j sum_d |q_d k_jd| / 8,
    the scale of the error of a score summed in fp32."""
    D = heads * 64
    x = qkv.double()
    out = torch.zeros(x.shape[0], D, dtype=torch.float64, device=x.device)
    mag, amp = torch.zeros_like(out), torch.zeros_like(out)
    for s in range(len(cu) - 1):
        a, b = cu[s], cu[s + 1]
        if b <= a:
            continue
        q = x[a:b, :D].view(b - a, heads, 64).transpose(0, 1)
        k = x[a:b, D:2 * D].view(b - a, heads, 64).transpose(0, 1)
        v = x[a:b, 2 * D:].view(b - a, heads, 64).transpose(0, 1)
        p = torch.softmax(q @ k.transpose(1, 2) / 8.0, dim=-1)
        out[a:b] = (p @ v).transpose(0, 1).reshape(b - a, D)
        mag[a:b] = (p @ v.abs()).transpose(0, 1).reshape(b - a, D)
        top = (q.abs() @ k.abs().transpose(1, 2) / 8.0).amax(-1)                 # [heads, len]
        amp[a:b] = top.T[:, :, None].expand(-1, -1, 64).reshape(b - a, D)
    return out, mag, amp


# ---- transformer stack: one layer of mer_run_stack (encoder.cu) ---------------------------------------------------------
# stack_layer restates one layer in float64 from the GPU's own input hidden state, with an elementwise bound built from
# the pieces above (the lambda = 4 model of the front end).  The stack stores its operands (LN outputs, q | k | v, ctx, the
# FC1 output) as fp16, tf32 or split bf16; each such store rounds by at most out_rounding(v), and that rounding enters
# the bound as LAMBDA * out_rounding(v): its standard deviation is at most out_rounding(v), and it is the dominant error
# of every layer, carried through the next linear stage in quadrature (_lin_err).  Stage by stage (encoder.cu):
#   LN          _ln_err (mer_layernorm_launch; pre-LN: LN1 / LN2 then the operand store; post-LN: fp32 x, then its copy)
#   linear      _lin_err with u_op = 0 for fp16 or tf32 operands (fp16- / tf32-exact weights and activations: exact
#               products), 2^-16 for split bf16 (hi hi + hi lo + lo hi; the dropped lo lo is <= 2^-16 |a| |w|); + u |z|
#               for the fp32 bias / residual add of the epilogue (linear() of encoder.cu, gemm.cu epilogue)
#   attention   _attention_err: the kernel's own (2^-11 + 16 u A + 8 u) P |V| (P rounded to fp16 or tf32 for P V in every
#               route), plus the q | k | v errors carried through softmax; a one-token row is exactly its v
#   activation  _gelu_err (gelu_erf_fast) or _quick_gelu_err (quick_gelu_fast), gemm.cu epi_act
# The input operand is applied exactly: post-LN layers read fp16(x) (MER_LN_SPLIT_F16) or split_bf16(x) of the previous
# LayerNorm's fp32 output, which is the hidden state itself.
STACK_UNIT = {None: 0.0, "f16": 0.0, "tf32": 0.0, "bf16x3": 2.0 ** -16}
STACK_OPERAND = {None: None, "f16": "f16", "tf32": "tf32", "bf16x3": "split"}
ATT_KERNEL = {"short": "attention_short_kernel", "f16": "attention_vt_kernel<true", "long": "attention_vt_kernel<true",
              "tc": "attention_vt_kernel<false", "fallback": "attention_kernel"}


def stack_route(mode, max_seqlen, long_rows=False):
    """Attention route of mer_run_stack for a stack in `mode` ("f16", "tf32", "bf16x3") whose batch has `max_seqlen`
    (encoder.cu: f16_long / f16_rows / long_att; attention.cu mer_attention_uses_tc; attention_f16.cu
    mer_attention_f16_supported; attention_short.cu mer_attention_short_enabled without MER_ATT_SHORT): "short" (fp16
    q | k | V^T, attention_short.cu, 129 .. 208 tokens), "f16" (fp16 q | k | V^T, tiled),
    "long" (the same kernel past 505 tokens, long_rows only), "tc" (tf32 q | k | V^T) or "fallback" (tf32 q | k | v read
    by attention.cu; an fp16 stack casts its fp32 context to fp16)."""
    tc = max_seqlen <= 253
    f16_long = long_rows and 505 < max_seqlen <= 4096
    f16_rows = f16_long or max_seqlen <= 505
    if mode == "f16":
        if f16_rows:
            return "short" if 128 < max_seqlen <= 208 else ("long" if f16_long else "f16")
        return "fallback"
    if not tc and f16_rows:
        return "long" if f16_long else "f16"
    return "tc" if tc else "fallback"


def stack_form(mode, pre_ln, max_seqlen, long_rows=False, quick=False, eps=1e-12, heads=12):
    return dict(mode=mode, pre_ln=pre_ln, route=None if mode is None else stack_route(mode, max_seqlen, long_rows),
                act="quick" if quick else "erf", eps=eps, heads=heads)


def packed_layer(pk, layers, l, mode):
    """Layer l's weights exactly as the encoder packed them on the device (MerLayerWeights pointers resolved through the
    Packed store): fp16 weights as stored (F16), the tf32-rounded copies (TF32), hi + lo of the split rows (BF16X3);
    LayerNorm parameters and biases fp32.  float64 tensors on the device."""
    by_ptr = {t.data_ptr(): t for t in pk.tensors}
    out = {}
    for name, _ in type(layers[l])._fields_:
        t = by_ptr[getattr(layers[l], name)]
        if name.startswith("w_") and mode == "bf16x3":
            hi, lo = split_halves(t)
            t = hi.double() + lo.double()
        out[name] = t.double()
    return out


def layer_from_state_dict(sd, names, l, device="cpu"):
    """The same dict from an HF state dict (float64, no operand rounding): q | k | v concatenated as pack_layers does."""
    g = lambda role: torch.as_tensor(np.asarray(sd[names[role].format(i=l)])).to(device, torch.float64)  # noqa: E731
    return dict(ln1_g=g("ln1_g"), ln1_b=g("ln1_b"), w_qkv=torch.cat([g("q_w"), g("k_w"), g("v_w")]),
                b_qkv=torch.cat([g("q_b"), g("k_b"), g("v_b")]), w_o=g("o_w"), b_o=g("o_b"), ln2_g=g("ln2_g"),
                ln2_b=g("ln2_b"), w_fc1=g("fc1_w"), b_fc1=g("fc1_b"), w_fc2=g("fc2_w"), b_fc2=g("fc2_b"))


def quick_gelu(x):
    return x * torch.sigmoid(1.702 * x)


def _quick_gelu_err(z, e):
    """quick_gelu_fast (mer_common.cuh): x * rcp.approx(1 + ex2.approx(-1.702 log2(e) x)).  |q''| <= 0.9, so the carried
    error is |q'| e + 0.45 e^2.  Own error, relative to |q|: the product and the reciprocal (2 u), the exponent's
    argument rounded (u |t|, t = 2.46 x, moving 2^t by ln 2 u |t| = 1.70 u |x|) and ex2.approx (2 u), both scaled by
    1 - sigmoid (the share of 2^t in 1 + 2^t), and the sum 1 + 2^t (u)."""
    s = torch.sigmoid(1.702 * z)
    q = z * s
    slope = (s + 1.702 * z * s * (1 - s)).abs()
    own = U32 * q.abs() * (3 + (1 - s) * (2 + 1.702 * z.abs()))
    return q, slope * e + 0.45 * e * e + own + 1e-30


def _store(v, e, fmt, emulate):
    """The stack stores v as fmt (None: fp32): returns (value, bound)."""
    if fmt is None:
        return v, e
    if emulate:
        return operand(v, fmt).to(v.dtype), e
    return v, e + LAMBDA * out_rounding(v, fmt != "split")


def operand(v, fmt):
    """Value of fp32 v stored as fmt: "f16" (cvt.rn.satfinite), "tf32" (cvt.rna), "split" (hi + lo)."""
    if fmt is None:
        return v
    if fmt == "f16":
        return f16_satfinite(v).to(v.dtype)
    if fmt == "tf32":
        return round_tf32_ties_away(v.float()).to(v.dtype)
    hi, lo = split_bf16(v)
    return (hi.double() + lo.double()).to(v.dtype)


def _attention_err(qkv, e, cu, heads, scale=0.125, fault=None):
    """(ctx, bound) of the stack's attention on packed q | k | v with elementwise bounds e.  The kernel's own error is
    that of tests/test_attention_fp32_gpu.py (attention_packed's P |V| and A).  Carried errors: a v error reaches ctx
    through P (in quadrature); a score error ds_ij (q and k errors, in quadrature over the head's 64 columns, / 8) moves
    ctx by sum_j P_ij (ds_ij - sum_l P_il ds_il) v_j, at most 2 max_j ds_ij P |V|.  A one-token row is v itself."""
    D = heads * 64
    ctx, mag, amp = attention_packed(qkv, cu, heads)
    bound = (2.0 ** -11 + 16 * U32 * amp + 8 * U32) * mag
    x, e = qkv.double(), e.double()
    for s in range(len(cu) - 1):
        a, b = cu[s], cu[s + 1]
        if b - a == 1:
            bound[a:b] = e[a:b, 2 * D:]
            continue
        hv = lambda t, c: t[a:b, c * D:(c + 1) * D].reshape(b - a, heads, 64).transpose(0, 1)  # noqa: E731
        q, k, v = hv(x, 0), hv(x, 1), hv(x, 2)
        eq, ek, ev = hv(e, 0), hv(e, 1), hv(e, 2)
        p = torch.softmax(q @ k.transpose(1, 2) * 0.125, dim=-1)
        ds = torch.sqrt((eq * eq) @ (k * k).transpose(1, 2) + (q * q) @ (ek * ek).transpose(1, 2)) * 0.125
        carried = torch.sqrt((p * p) @ (ev * ev)) + 2 * ds.amax(-1, keepdim=True) * (p @ v.abs())
        bound[a:b] += carried.transpose(0, 1).reshape(b - a, D)
    if fault is not None:                   # tests of the bound only: a restatement of a wrong attention
        ctx = _faulty_attention(x, cu, heads, scale, fault)
    return ctx, bound


def _faulty_attention(x, cu, heads, scale, fault):
    D = heads * 64
    q, k, v = x[:, :D], x[:, D:2 * D], x[:, 2 * D:]
    if fault == "head_k":                   # head h reads head h + 1's keys
        k = torch.roll(k.view(-1, heads, 64), -1, dims=1).reshape(-1, D)
    if fault == "key_shift":                # a V^T column offset: token j reads token j + 1's value
        v = torch.roll(v, -1, dims=0)
    return attention_packed(torch.cat([q * (scale / 0.125), k, v], 1), cu, heads)[0]


def stack_layer(w, x_in, cu, form, fault=None, emulate=False, op_in=None, trace=None):
    """One layer of mer_run_stack on x_in [tokens, D] (the GPU's hidden state l) with packed cu_seqlens `cu` (a list),
    weights w (packed_layer / layer_from_state_dict) and `form` (stack_form).  Returns (x_out, bound): float64, or with
    `emulate` an fp32 evaluation that rounds every stored operand (bound None).  form["mode"] None: no operand rounding
    anywhere (the network itself, for the comparison with the oracle).
    For the tests of the bound only: `fault` restates a wrong layer (see STACK_FAULTS); op_in replaces the input operand
    copy of a post-LN layer; trace (a dict) receives the post-LN layer's fp32 x after LN1 as trace["x1"]."""
    dt = torch.float32 if emulate else torch.float64
    x = x_in.to(dt)
    fmt = STACK_OPERAND[form["mode"]]
    u_op = STACK_UNIT[form["mode"]]
    route = form["route"]
    qkv_fmt = None if fmt is None else ("f16" if route in ("short", "f16", "long") else "tf32")
    D, eps, heads = x.shape[-1], form["eps"], form["heads"]
    pre_ln = form["pre_ln"] != (fault == "ln_order")
    W = {k: v.to(dt) for k, v in w.items()}
    if fault == "ln_swap":
        for a, b in (("ln1_g", "ln2_g"), ("ln1_b", "ln2_b")):
            W[a], W[b] = W[b], W[a]
    for name in ("b_qkv", "b_o", "b_fc1", "b_fc2", "ln1_b", "ln2_b"):
        if fault == "drop_" + name:
            W[name] = torch.zeros_like(W[name])
    zero = torch.zeros_like(x)

    def ln(v, ev, g, b):
        if emulate:
            return F.layer_norm(v, (D,), g, b, eps), None
        return _ln_err(v, ev, g, b, eps)

    def lin(a, ea, wname, bname, res=None, eres=None):
        z = a @ W[wname].T + W[bname]
        if res is not None:
            z = z + res
        if emulate:
            return z, None
        e = _lin_err(lambda t, ww: t @ ww.T, a, ea, W[wname], u_op, a.shape[-1]) + U32 * z.abs()
        return z, e if eres is None else e + eres

    if pre_ln:
        a, ea = _store(*ln(x, zero, W["ln1_g"], W["ln1_b"]), fmt, emulate)
    else:
        a = operand(x if op_in is None else op_in.to(dt), fmt)
        ea = None if emulate else zero
    qkv, eqkv = _store(*lin(a, ea, "w_qkv", "b_qkv"), qkv_fmt, emulate)
    scale = 1.0 / math.sqrt(D) if fault == "scale" else 0.125
    att_fault = fault if fault in ("scale", "head_k", "key_shift") else None
    if emulate:
        ctx = _emulated_attention(qkv, cu, heads, "f16" if route in ("short", "f16", "long") else "tf32")
        ectx = None
    else:
        ctx, ectx = _attention_err(qkv, eqkv, cu, heads, scale, att_fault)
    ctx, ectx = _store(ctx, ectx, fmt, emulate)     # the fp16 fallback's mer_cast_f16 is the same rounding
    res = None if fault == "no_residual" else x
    s, es = lin(ctx, ectx, "w_o", "b_o", res, None if emulate else zero)
    if pre_ln:
        x1, ex1 = s, es
        a2, ea2 = _store(*ln(x1, ex1, W["ln2_g"], W["ln2_b"]), fmt, emulate)
    else:
        x1, ex1 = ln(s, es, W["ln1_g"], W["ln1_b"])
        a2, ea2 = _store(x1, ex1, fmt, emulate)
    if trace is not None:
        trace["x1"] = x1
    z, ez = lin(a2, ea2, "w_fc1", "b_fc1")
    quick = (form["act"] == "quick") != (fault == "act")
    if emulate:
        h, eh = (quick_gelu(z) if quick else 0.5 * z * (1 + torch.erf(z / math.sqrt(2.0)))), None
    else:
        h, eh = (_quick_gelu_err if quick else _gelu_err)(z, ez)
    h, eh = _store(h, eh, fmt, emulate)
    s2, es2 = lin(h, eh, "w_fc2", "b_fc2", x1, ex1)
    if pre_ln:
        return s2, es2
    return ln(s2, es2, W["ln2_g"], W["ln2_b"])


STACK_FAULTS = ("act", "drop_b_qkv", "drop_b_o", "drop_b_fc1", "drop_b_fc2", "drop_ln1_b", "drop_ln2_b", "ln_swap",
                "ln_order", "scale", "head_k", "key_shift", "no_residual", "stale_operand")


def _emulated_attention(qkv, cu, heads, p_fmt):
    """fp32 attention with P rounded to p_fmt for the P V product (fp16 in the fp16 V^T kernels, tf32 ties-away in the
    tf32 V^T kernel and attention.cu), normalised by the fp32 sum of the unrounded P."""
    D = heads * 64
    x = qkv.float()
    out = torch.zeros(x.shape[0], D, dtype=torch.float32, device=x.device)
    for s in range(len(cu) - 1):
        a, b = cu[s], cu[s + 1]
        q, k, v = (x[a:b, c * D:(c + 1) * D].reshape(b - a, heads, 64).transpose(0, 1) for c in range(3))
        sc = q @ k.transpose(1, 2) * 0.125
        p = torch.exp(sc - sc.amax(-1, keepdim=True))
        pr = p.half().float() if p_fmt == "f16" else round_tf32_ties_away(p.contiguous())
        out[a:b] = ((pr @ v) / p.sum(-1, keepdim=True)).transpose(0, 1).reshape(b - a, D)
    return out


def biased_attention(qkv, bias, rowscale, batch, T, heads):
    """softmax_j((q_i / 8) . k_j + rowscale[b, i, h] * bias[h, i, j]) v_j.  Returns (ctx, P |V|, S): S is the row's score
    error in units of u for 64 chained fp32 FMAs and one more for the bias: 65 max_j sum_d |q_d k_jd| / 8 + max_j
    |rowscale * bias_ij|, the latter over the keys that keep a non-zero probability."""
    D = heads * 64
    x = qkv.double().view(batch, T, 3, heads, 64)
    q, k, v = (x[:, :, i].transpose(1, 2) for i in range(3))                    # [batch, heads, T, 64]
    s = (q * 0.125) @ k.transpose(2, 3)
    rs = 1.0 if rowscale is None else rowscale.double().view(batch, T, heads).permute(0, 2, 1)[..., None]
    add = rs * bias.double()[None]
    p = torch.softmax(s + add, dim=-1)
    top = 65 * ((q.abs() * 0.125) @ k.abs().transpose(2, 3)).amax(-1) + \
        (add.abs() * (p > 1e-30)).expand_as(p).amax(-1)                                      # [batch, heads, T]
    flat = lambda t: t.transpose(1, 2).reshape(batch * T, D)  # noqa: E731
    return flat(p @ v), flat(p @ v.abs()), flat(top[..., None].expand(-1, -1, -1, 64))


def wavlm_gate(x, w, b, c, heads):
    """gate = ga * (gb * c[head] - 1) + 2, (ga, gb) = sigmoid of the two 4-sums of w [8, 64] . x_head + b [8]."""
    t = x.double().view(-1, heads, 64) @ w.double().T + b.double()               # [tokens, heads, 8]
    ga, gb = torch.sigmoid(t[..., :4].sum(-1)), torch.sigmoid(t[..., 4:].sum(-1))
    return ga * (gb * c.double()[None] - 1.0) + 2.0


def small_attention(q, k, v, causal):
    """q [batch, nq, heads, 64], k / v [batch, nk, heads, 64] -> (out [batch, nq, heads, 64], P |V|, A [batch, nq, heads,
    1] = max_j sum_d |q_d k_jd| / 8 over the visible keys); under `causal` query i sees keys 0 .. i."""
    q, k, v = (t.double().transpose(1, 2) for t in (q, k, v))
    nq, nk = q.shape[2], k.shape[2]
    keep = torch.ones(nq, nk, dtype=torch.bool, device=q.device)
    if causal:
        keep = torch.arange(nk, device=q.device)[None, :] <= torch.arange(nq, device=q.device)[:, None]
        k, v = torch.nan_to_num(k, nan=0.0), torch.nan_to_num(v, nan=0.0)   # keys no query may see hold NaN in the tests
    s = (q @ k.transpose(2, 3) / 8.0).masked_fill(~keep, float("-inf"))
    p = torch.softmax(s, dim=-1)
    top = (q.abs() @ k.abs().transpose(2, 3) / 8.0).masked_fill(~keep, 0.0).amax(-1, keepdim=True)
    return (p @ v).transpose(1, 2), (p @ v.abs()).transpose(1, 2), top.transpose(1, 2)


def swiglu(x, hidden):
    x = x.double()
    a, b = x[:, :hidden], x[:, hidden:]
    return a * torch.sigmoid(a) * b


def videomae_patches(frames_bgr, mean, std):
    """The layout mer_videomae_patchify writes: rows = (clip, tubelet, patch row, patch column), K = (channel RGB,
    frame in tubelet, dy, dx); values (pix / 255 - mean) / std."""
    n = frames_bgr.shape[0] // 16
    x = frames_bgr.flip(-1).double() / 255.0
    x = (x - torch.tensor(mean, dtype=torch.float64, device=x.device)) / torch.tensor(std, dtype=torch.float64,
                                                                                      device=x.device)
    x = x.reshape(n, 8, 2, 14, 16, 14, 16, 3).permute(0, 1, 3, 5, 7, 2, 4, 6)    # n, tt, py, px, c, dt, dy, dx
    return x.reshape(n * 1568, 1536)


# ---- fusion nets: dropout hash, float64 loss / gradients, Adam -------------------------------------------------------
_M64 = (1 << 64) - 1


def keep_mask(seed, m, step, n, p):
    """Elements 0 .. n-1 of keep-mask tensor m at step counter `step` as the fusion kernels draw them, as a bool numpy
    array: keep_hash of fusion_fused.cu (seed + 0x1000 (m + 1) + 0x9E37.. (step + 1) + 0xD1B5.. (i + 1), the splitmix64
    finaliser, u = top 24 bits / 2^24, keep when u >= p in fp32).  m = None is fus_dropout_mask_kernel's form of fusion.cu,
    whose seed already carries the tensor's 0x1000 (m + 1)."""
    base = (int(seed) + (0 if m is None else 0x1000 * (m + 1)) + 0x9E3779B97F4A7C15 * (int(step) + 1)) & _M64
    z = np.arange(1, n + 1, dtype=np.uint64) * np.uint64(0xD1B54A32D192ED03) + np.uint64(base)  # wraps mod 2^64
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z ^= z >> np.uint64(31)
    u = (z >> np.uint64(40)).astype(np.float32) * np.float32(2.0 ** -24)
    return u >= np.float32(p)


def keep_probability(p):
    """Exact keep probability of keep_mask: u takes the 2^24 values k / 2^24, and u >= p for all but ceil(p 2^24)."""
    return 1.0 - math.ceil(float(np.float32(p)) * 2 ** 24) / 2 ** 24


def fusion_f64(sd, inputs, p=0.0, masks=None, emo=None, val=None, upstream=None):
    """The fusion net in float64 through the oracle's own dtype-generic forward (oracle/fusion.py): Attention when `inputs`
    is (audios, texts, videos) with a state dict of audio_encoder.* keys (utterance or frame level), Attention_TOPN when
    the state dict has encoder0.* keys and `inputs` is the list of features.  Parameters, inputs and keep-masks are double
    copies of what the kernels read.  Returns dict(out=(features, emos, vals), and with emo / val: loss=(ce, mse, total)
    and grads={name: d total / d param}; with upstream=(w_features, w_emos, w_vals): up={name: d sum(out * w) / d param})."""
    from oracle import fusion as OF
    dev = inputs[0].device
    sd64 = {k: torch.as_tensor(v).to(dev, torch.float64).requires_grad_(True) for k, v in sd.items()}
    xs = [x.to(torch.float64) for x in inputs]
    mk = None if masks is None else [None if mm is None else torch.as_tensor(mm).to(dev, torch.float64) for mm in masks]
    if "encoder0.linear_1.weight" in sd64:
        out = OF.attention_topn_forward(sd64, xs, mk, p)
    else:
        out = OF.attention_forward(sd64, *xs, masks=mk, p=p)
    res = dict(out=tuple(o.detach() for o in out))
    names, leaves = list(sd64), list(sd64.values())
    if emo is not None:
        ce, mse = OF.losses(out[1], out[2], emo.to(dev), val.to(dev, torch.float64))
        total = ce + mse
        g = torch.autograd.grad(total, leaves, retain_graph=upstream is not None, allow_unused=True)
        res["loss"] = tuple(float(x.detach()) for x in (ce, mse, total))
        res["grads"] = {n: torch.zeros_like(x) if gi is None else gi for n, x, gi in zip(names, leaves, g)}
    if upstream is not None:
        s = sum((o * w.to(torch.float64)).sum() for o, w in zip(out, upstream))
        g = torch.autograd.grad(s, leaves, allow_unused=True)
        res["up"] = {n: torch.zeros_like(x) if gi is None else gi for n, x, gi in zip(names, leaves, g)}
    return res


def adam_f64(param, grad, exp_avg, exp_avg_sq, t, lr, beta1, beta2, eps, weight_decay, grad_scale=1.0, clip=0.0):
    """torch.optim.Adam(lr, (beta1, beta2), eps, weight_decay) step t (1-based) in float64, after clip_grad_value_(clip)
    (clip > 0) of grad * grad_scale; coupled L2 (weight_decay * param added to the clipped gradient).  The hyper-
    parameters are taken at their fp32 values, as the kernels receive them.  Returns (param, exp_avg, exp_avg_sq)."""
    h = [float(np.float32(x)) for x in (lr, beta1, beta2, eps, weight_decay, grad_scale, clip)]
    lr, beta1, beta2, eps, weight_decay, grad_scale, clip = h
    p, g, m, v = (x.to(torch.float64) for x in (param, grad, exp_avg, exp_avg_sq))
    g = g * grad_scale
    if clip > 0:
        g = g.clamp(-clip, clip)
    g = g + weight_decay * p
    m = beta1 * m + (1.0 - beta1) * g
    v = beta2 * v + (1.0 - beta2) * g * g
    denom = v.sqrt() / math.sqrt(1.0 - beta2 ** t) + eps
    return p - lr / (1.0 - beta1 ** t) * m / denom, m, v


# ---- table-driven CNN executor (mer_cnn_forward, resnet.cu) -----------------------------------------------------------
# GEMM operand formats.  MER_GEMM_F16 converts each fp32 activation with cvt.rn.satfinite (round to nearest even, clamp
# to +-65504, NaN stays NaN); MER_GEMM_BF16X3 stores hi = bf16(x) and lo = bf16(x - hi) (both round to nearest even)
# and its MMAs add hi hi + hi lo + lo hi: the lo lo product is left out (tests/test_gemm_gpu.py).
GEMM_F16, GEMM_BF16X3 = 2, 1


def f16_satfinite(x):
    """cvt.rn.satfinite.f16.f32 on fp32 values, returned as fp32."""
    return x.float().clamp(-65504.0, 65504.0).half().float()


def split_bf16(x):
    """(hi, lo) of the split-bf16 operand of fp32 values: hi = RNE bf16 of x, lo = RNE bf16 of x - hi (exact in fp32)."""
    x = x.float()
    hi = round_bf16_nearest_even(x)
    return hi, round_bf16_nearest_even(x - hi)


def stem_operand(frames_bgr, scale, mean, std):
    """The value im2col_stem_kernel computes for each pixel, bit for bit: fma(pix, scale, -mean[c]) rounded once to fp32
    (pix * scale is exact in float64 for 8-bit pixels and an fp32 scale, and so is its difference with an fp32 mean),
    then an IEEE fp32 division by std[c]; channels in RGB order (BGR input).  frames: uint8 [n, H, W, 3] -> fp32."""
    f32 = lambda v: torch.tensor([float(np.float32(t)) for t in v], dtype=torch.float64)  # noqa: E731
    pix = torch.as_tensor(np.ascontiguousarray(np.asarray(frames_bgr)[..., ::-1])).double()
    num = (pix * float(np.float32(scale)) - f32(mean)).float()
    return num / f32(std).float()


def cnn_conv(x, w, b, k, stride, pad, mode=None, res=None):
    """NHWC convolution of the operand values of x [n, H, W, cin] with w [cout_pad, >= k k cin] in (ky, kx, c) order
    and bias b, in float64: mode None computes on x and w as given, GEMM_F16 on their satfinite fp16 values,
    GEMM_BF16X3 on split operands without the lo lo product.  Returns (y, a): a = |x| |w| + |b| (+ |res|) on the same
    operands, the scale the GEMM's accumulation error is measured against."""
    x, w = x.float(), torch.as_tensor(w).float()
    cin, co = x.shape[-1], w.shape[0]
    kk = k * k * cin
    wt = lambda v: v[:, :kk].reshape(co, k, k, cin).permute(0, 3, 1, 2).double()  # noqa: E731
    cv = lambda v, ww: F.conv2d(v.permute(0, 3, 1, 2).double(), ww, stride=stride, padding=pad)  # noqa: E731
    if mode == GEMM_BF16X3:
        (xh, xl), (wh, wl) = split_bf16(x), split_bf16(w)
        y = cv(xh, wt(wh) + wt(wl)) + cv(xl, wt(wh))
        a = cv(xh.abs(), wt(wh).abs() + wt(wl).abs()) + cv(xl.abs(), wt(wh).abs())
    else:
        if mode == GEMM_F16:
            x, w = f16_satfinite(x), f16_satfinite(w)
        y, a = cv(x, wt(w)), cv(x.abs(), wt(w).abs())
    b = torch.as_tensor(b).double()
    y, a = (y + b[:, None, None]).permute(0, 2, 3, 1), (a + b.abs()[:, None, None]).permute(0, 2, 3, 1)
    if res is not None:
        assert tuple(res.shape) == tuple(y.shape), f"residual {tuple(res.shape)} for an output {tuple(y.shape)}"
        y, a = y + res.double(), a + res.double().abs()
    return y, a


def cnn_plan(m, n):
    """Workspace layout of mer_cnn_forward for an op table (cnn_walk's planning pass): per buffer the largest
    n H W Cs fp32 map any op defines there, each 256-byte aligned in index order, then the im2col operand, the
    average pool's offsets and the SE means and gates.  Returns (dict of byte offsets and total, {buffer: (H, W, C,
    Cs)} as the last op left them)."""
    al = lambda v: (v + 255) & ~255  # noqa: E731
    vb = 4 if m.gemm_mode == GEMM_BF16X3 else 2
    sh, need, col, se_c = {}, [0] * 24, 0, 0

    def define(bi, s):
        sh[bi] = s
        need[bi] = max(need[bi], n * s[0] * s[1] * s[3])
    for i in range(m.n_ops):
        op = m.ops[i]
        p = [op.p[j] for j in range(4)]
        if op.kind == 0:                                                             # STEM
            c = m.convs[op.conv]
            oh, ow = (m.in_h - 1) // 2 + 1, (m.in_w - 1) // 2 + 1
            col = max(col, n * oh * ow * c.kpad * vb)
            define(op.dst, (oh, ow, c.cout, c.cout_pad))
        elif op.kind == 1:                                                           # CONV
            c, s = m.convs[op.conv], sh[op.src]
            oh, ow = (s[0] + 2 * c.pad - c.k) // c.stride + 1, (s[1] + 2 * c.pad - c.k) // c.stride + 1
            col = max(col, n * oh * ow * c.kpad * vb)
            define(op.dst, (oh, ow, c.cout, c.cout_pad))
        elif op.kind == 2:                                                           # MAXPOOL
            s = sh[op.src]
            if op.k == 2:
                define(op.dst, (s[0] // 2, s[1] // 2, s[2], s[3]))
            else:
                po = [pool_out_size(v, op.pad, op.ceil_mode) for v in s[:2]]
                define(op.dst, (po[0], po[1], s[2], s[3]))
        elif op.kind in (4, 8):                                                      # SE, CBAM
            if op.kind == 4:
                se_c = max(se_c, sh[op.src][2])
            define(op.dst, sh[op.src])
        elif op.kind == 5:                                                           # CROP
            s = sh[op.src]
            define(op.dst, (p[2], p[3], s[2], s[3]))
        elif op.kind == 6:                                                           # SHAPE
            s = sh[op.src]
            define(op.dst, (s[0], s[1], p[0], p[0]))
        elif op.kind == 9:                                                           # AFFINE
            s, c = sh[op.src], m.convs[op.conv].cout
            define(op.dst, (s[0], s[1], c, c))
        elif op.kind == 10:                                                          # UPADD
            define(op.dst, sh[op.res])
    off, o = {}, 0
    for bi in range(24):
        off[bi] = o
        o += al(need[bi] * 4)
    for name, size in (("col", col), ("cu", (n + 1) * 4), ("z", n * se_c * 4), ("scale", n * se_c * 4)):
        off[name] = o
        o += al(size)
    off["total"] = o
    return off, sh


def pool_out_size(v, pad, ceil_mode):
    """torch MaxPool2d(3, 2, pad, ceil_mode) output length (aten pooling_output_shape); < 1 where torch raises."""
    o = (v + 2 * pad - 3 + (1 if ceil_mode else 0)) // 2 + 1
    if ceil_mode and (o - 1) * 2 >= v + pad:
        o -= 1
    return o


def interpret_cnn_tables(m, store, frames_bgr=None, dtype=torch.float32, bufs=None, operands=False):
    """Interpreter of a mer_cnn_forward op table (include/mer_b200.h: MerCnnOp) with the buffer / shape semantics of
    resnet.cu's executor, on NHWC maps with padded channel counts, in `dtype`.  store maps the w / b addresses of the
    table's MerResnetConv entries to their fp32 values (numpy or torch).  bufs: {index: [n, H, W, Cs] tensor} of
    buffer contents to start from (what a test wrote into the workspace; a SHAPE op keeps a buffer given here).
    operands: convolutions compute on the GEMM operands of m.gemm_mode (cnn_conv) and the stem on stem_operand, as
    the kernels do; otherwise on the exact values (the network's own semantics).
    Returns (out_feats [n, feat_dim], {index: tensor} of every buffer as the last op left it)."""
    n = len(frames_bgr) if frames_bgr is not None else next(iter(bufs.values())).shape[0]
    T = lambda v: torch.as_tensor(np.asarray(v, np.float32)).to(dtype)  # noqa: E731
    mode = m.gemm_mode if operands else None
    buf = {i: v.to(dtype).clone() for i, v in (bufs or {}).items()}
    real = {i: v.shape[-1] for i, v in buf.items()}
    given = set(buf)
    out = torch.full((n, m.feat_dim), float("nan"), dtype=dtype)
    mean, std = [m.mean[i] for i in range(3)], [m.std[i] for i in range(3)]

    def conv(x, c, res=None):
        kk = c.k * c.k * c.cin
        assert c.kpad == kk or (c.cin == 3 and c.kpad in (160, 192))
        return cnn_conv(x, T(store[c.w]), T(store[c.b]), c.k, c.stride, c.pad, mode, res)[0].to(dtype)
    for i in range(m.n_ops):
        op = m.ops[i]
        p = [op.p[j] for j in range(4)]
        res = buf[op.res] if op.res >= 0 and op.kind in (0, 1) else None
        if op.kind == 0:                                                             # STEM
            c = m.convs[op.conv]
            if operands:
                x0 = stem_operand(frames_bgr, m.scale, mean, std)
            else:
                pix = torch.as_tensor(np.ascontiguousarray(np.asarray(frames_bgr)[..., ::-1])).to(dtype)
                x0 = (pix * m.scale - torch.tensor(mean, dtype=dtype)) / torch.tensor(std, dtype=dtype)
            y = conv(x0, c, res)
            buf[op.dst], real[op.dst] = (torch.relu(y) if op.relu else y), c.cout
        elif op.kind == 1:                                                           # CONV
            c = m.convs[op.conv]
            assert op.src != op.dst and p[0] + c.cin <= real[op.src]
            y = conv(buf[op.src][..., p[0]:p[0] + c.cin], c, res)
            buf[op.dst], real[op.dst] = (torch.relu(y) if op.relu else y), c.cout
        elif op.kind == 2:                                                           # MAXPOOL
            assert op.k in (2, 3) and op.stride == 2 and op.src != op.dst
            xin = buf[op.src].permute(0, 3, 1, 2)
            y = F.max_pool2d(xin, 2, 2) if op.k == 2 else F.max_pool2d(xin, 3, 2, op.pad, ceil_mode=bool(op.ceil_mode))
            buf[op.dst], real[op.dst] = y.permute(0, 2, 3, 1), real[op.src]
        elif op.kind == 9:                                                           # AFFINE
            af = m.convs[op.conv]
            v = buf[op.src][..., p[0]:p[0] + af.cout] * T(store[af.w]) + T(store[af.b])
            assert op.src != op.dst
            buf[op.dst], real[op.dst] = (torch.relu(v) if op.relu else v), af.cout
        elif op.kind == 10:                                                          # UPADD
            up = buf[op.src].repeat_interleave(2, dim=1).repeat_interleave(2, dim=2)
            buf[op.dst], real[op.dst] = buf[op.res] + up, real[op.res]
        elif op.kind == 11:                                                          # MASKMUL
            mask = buf[op.res][..., :p[3]].sum(dim=3, keepdim=True)
            buf[op.dst][..., p[1]:p[1] + p[2]] = buf[op.src][..., p[0]:p[0] + p[2]] * mask
        elif op.kind == 4:                                                           # SE
            dn, up = m.convs[op.conv], m.convs[op.k]
            y = buf[op.src]
            d = torch.relu(y.mean(dim=(1, 2)) @ T(store[dn.w]).T + T(store[dn.b]))
            g = torch.sigmoid(d @ T(store[up.w]).T + T(store[up.b]))
            buf[op.dst], real[op.dst] = torch.relu(g[:, None, None, :] * y + buf[op.res]), real[op.src]
        elif op.kind == 5:                                                           # CROP
            buf[op.dst], real[op.dst] = buf[op.src][:, p[0]:p[0] + p[2], p[1]:p[1] + p[3]].clone(), real[op.src]
        elif op.kind == 6:                                                           # SHAPE
            if op.dst not in given:
                hh, ww = buf[op.src].shape[1:3]
                buf[op.dst] = torch.full((n, hh, ww, p[0]), float("nan"), dtype=dtype)
            real[op.dst] = p[0]
        elif op.kind == 7:                                                           # SLICE
            v = buf[op.src][..., p[0]:p[0] + p[2]]
            v = torch.relu(v) if op.relu == 1 else v
            if op.res >= 0:
                v = v + buf[op.res][..., p[3]:p[3] + p[2]]
            buf[op.dst][..., p[1]:p[1] + p[2]] = torch.relu(v) if op.relu == 2 else v
        elif op.kind == 8:                                                           # CBAM
            l1, l2, sp = m.convs[op.conv], m.convs[p[0]], m.convs[p[1]]
            y = buf[op.src]
            assert y.shape[-1] == real[op.src] == l1.cin

            def mlp(v):
                return torch.relu(v @ T(store[l1.w]).T + T(store[l1.b])) @ T(store[l2.w]).T + T(store[l2.b])
            y1 = y * torch.sigmoid(mlp(y.mean(dim=(1, 2))) + mlp(y.amax(dim=(1, 2))))[:, None, None, :]
            comp = torch.stack((y1.amax(dim=3), y1.mean(dim=3)), dim=1)              # [n, 2, H, W]: max, mean
            sg = torch.sigmoid(F.conv2d(comp, T(store[sp.w]).reshape(1, 2, 7, 7), T(store[sp.b]), padding=3))
            buf[op.dst], real[op.dst] = torch.relu(y1 * sg[:, 0, :, :, None] + buf[op.res]), real[op.src]
        else:
            assert op.kind == 3                                                      # GAP
            v = buf[op.src][..., :real[op.src]].mean(dim=(1, 2)) / max(p[2], 1)
            cols = slice(p[0], p[0] + real[op.src])
            out[:, cols] = out[:, cols] + v if p[1] else v
    return out, buf


def cnn_model(convs, ops, gemm_mode, in_hw, feat_dim, scale=1.0, mean=(0.0, 0.0, 0.0), std=(1.0, 1.0, 1.0)):
    """A MerCnnModel from plain lists: convs of dicts of MerResnetConv fields, ops of dicts of MerCnnOp fields (missing
    ones: conv / res -1, src / dst 0, the rest 0).  Returns (model, keep-alive list)."""
    import ctypes as C

    from mertools_b200 import encoders as En
    ca = (En.MerResnetConv * len(convs))()
    for c, d in zip(ca, convs):
        for k, v in d.items():
            setattr(c, k, v)
    oa = (En.MerCnnOp * len(ops))()
    for o, d in zip(oa, ops):
        o.conv, o.res = -1, -1
        for k, v in d.items():
            if k == "p":
                o.p = (C.c_int * 4)(*(list(v) + [0] * (4 - len(v))))
            else:
                setattr(o, k, v)
    m = En.MerCnnModel()
    m.convs, m.n_convs, m.ops, m.n_ops = ca, len(convs), oa, len(ops)
    m.gemm_mode, (m.in_h, m.in_w), m.scale, m.feat_dim = gemm_mode, in_hw, scale, feat_dim
    m.mean, m.std = (C.c_float * 3)(*mean), (C.c_float * 3)(*std)
    return m, [ca, oa]


def cnn_refused_tables(w=0x7F0000000000, b=0x7F0000001000):
    """(name, model, keep-alive, expected mer_last_error fragment) of op tables the executor cannot run: each would
    launch the stem's gather (and GEMM) before conv() or mer_gemm_launch refused it, so the planning pass refuses them.
    Every convolution entry points at w and b: the default addresses are never dereferenced while the planner refuses
    these tables on a machine without a GPU; a GPU test passes real zeroed buffers (>= 192 * 192 * 4 bytes for w,
    >= 192 * 4 for b) so that a table wrongly accepted runs on readable memory and fails on its launch count."""
    from mertools_b200 import _lib as L

    def conv(cin, cout, cout_pad, k, stride, pad, kpad=None):
        return dict(w=w, b=b, cin=cin, cout=cout, cout_pad=cout_pad, k=k, stride=stride, pad=pad,
                    kpad=k * k * cin if kpad is None else kpad)
    stem = conv(3, 64, 128, 7, 2, 3, 192)
    stem_s = conv(3, 64, 128, 7, 2, 3, 160)
    shape = lambda c: [dict(kind=6, src=0, dst=1, p=(c,))]  # noqa: E731
    F16, BF = L.MER_GEMM_F16, L.MER_GEMM_BF16X3
    # (name, gemm mode, frame h x w, convs, ops between the stem and the GAP, expected message); a frame of 3 x 3
    # gives a 2 x 2 stem output, 1 x 1 a 1 x 1 one.  With a second conv entry the table ends in CONV 1 -> 2 + GAP 2,
    # otherwise in a GAP of the last op's dst.
    cases = [
        # f16 3x3 over 32 channels: K = 288 is no multiple of the f16 GEMM's 64-wide K step
        ("f16 K 288", F16, (3, 3), [stem, conv(32, 128, 128, 3, 1, 1)], shape(32), "conv geometry"),
        ("split K 72", BF, (3, 3), [stem_s, conv(8, 128, 128, 3, 1, 1)], shape(8), "conv geometry"),
        ("kpad != k k cin", F16, (3, 3), [stem, conv(64, 128, 128, 1, 1, 0, kpad=128)], shape(64), "conv geometry"),
        ("cin % 8", BF, (3, 3), [stem_s, conv(4, 128, 128, 4, 1, 0)], shape(4), "conv geometry"),
        ("cout_pad % 128", F16, (3, 3), [stem, conv(64, 64, 64, 1, 1, 0)], shape(64), "conv geometry"),
        ("cout > cout_pad", F16, (3, 3), [stem, conv(64, 256, 128, 1, 1, 0)], shape(64), "conv geometry"),
        ("stride 0", F16, (3, 3), [stem, conv(64, 128, 128, 1, 0, 0)], shape(64), "conv geometry"),
        ("k 0", F16, (3, 3), [stem, conv(64, 128, 128, 0, 1, 0, kpad=0)], shape(64), "conv geometry"),
        ("7x7 of a 2 x 2 map", F16, (3, 3), [stem, conv(64, 128, 128, 7, 1, 0)], shape(64),
         "conv (pad 0) of a 2 x 2 map"),
        ("stem cout_pad 192", F16, (3, 3), [conv(3, 64, 192, 7, 2, 3, 192)], [], "stem geometry"),
        ("stem cout > cout_pad", F16, (3, 3), [conv(3, 256, 128, 7, 2, 3, 192)], [], "stem geometry"),
        ("3x3/2 pool pad 0 of 1 x 1", F16, (1, 1), [stem], [dict(kind=2, src=0, dst=1, k=3, stride=2, pad=0)],
         "max-pool (pad 0) of a 1 x 1 map"),
        ("3x3/2 floor pool pad 0 of 2 x 2", F16, (3, 3), [stem],
         [dict(kind=5, src=0, dst=2, p=(0, 0, 2, 2)), dict(kind=2, src=2, dst=1, k=3, stride=2, pad=0)],
         "max-pool (pad 0) of a 2 x 2 map"),
        ("3x3/2 pool pad 2", F16, (3, 3), [stem], [dict(kind=2, src=0, dst=1, k=3, stride=2, pad=2)], "max-pool (pad 2)"),
    ]
    out = []
    for name, mode, hw, convs, mid, msg in cases:
        ops = [dict(kind=0, conv=0, dst=0, relu=1)] + mid
        if len(convs) > 1:
            ops += [dict(kind=1, conv=1, src=1, dst=2), dict(kind=3, src=2)]
        else:
            ops.append(dict(kind=3, src=ops[-1]["dst"]))
        m, keep = cnn_model(convs, ops, mode, hw, 256)
        out.append((name, m, keep, msg))
    return out
