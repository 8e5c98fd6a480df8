"""float64 restatements of the row-wise and fp32 attention entry points of include/mer_b200.h, of the fusion nets'
dropout hash, loss, gradients and Adam, and the small helpers the kernel-level GPU tests share (environment switches,
guarded output buffers).  Every function takes torch tensors on any device and computes in float64 on that device;
tests/test_kernel_refs.py checks them on the CPU against torch's own operators."""
import contextlib
import math
import os

import numpy as np
import torch

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
