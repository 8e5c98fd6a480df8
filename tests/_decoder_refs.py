"""float64 restatements of one layer of the host-orchestrated decoder text stacks (extract/llama_text.py: LLaMA;
extract/ln_decoder_text.py: BLOOM, OPT, GPT-2, Falcon), with elementwise error bounds of the CUDA path, in the style of
stack_layer (tests/_kernel_refs.py).  Every function computes in float64 on its inputs' device.

Weights are restated from the HF-named state dict (synthetic.*_state_dict, or a full-width dict of the same names),
rounded to fp16 as the loader rounds them, and laid out here in HF's own terms: BLOOM's fused query_key_value read as
[head][q, k, v][head_dim] rows (BloomAttention._split_heads), Falcon's as heads x q | one k | one v head, GPT-2's Conv1D
weights as [in, out] with c_attn's columns q | k | v, OPT's and LLaMA's separate projections.  None of the packed layer
dicts of the nets is read, so deinterleave_qkv, falcon_qkv / falcon_out, the Conv1D transpose and the q | k | v
concatenation stay under test.  The exception: the rotary cos / sin operands are rope_tables' fp32 values (compared
with HF's construction in tests/test_decoder_refs.py), and BLOOM's slopes alibi_slopes' fp32 values.

Bounds (u = 2^-24; LAMBDA, _lin_err, out_rounding and attention_tc_bound as in tests/_kernel_refs.py).  The layer is fed
the GPU's own fp32 hidden state, so its input carries no error; each stage carries the error of its inputs and adds its
own:
  RMSNorm     y = w (x r), r = rsqrtf(ss / D + eps), ss an fp32 fma chain of D / 256 squares per thread, then 5
              shuffle and 8 shared-memory adds: ss relative (D / 256 + 13) u; r half of it, + 2 ulp rsqrtf, + the
              division and the eps add; the two products 2 u: own (D / 512 + 12) u |y|.  Carried: the gain |w| / rms
              (the rest of the derivative is an orthogonal projection, which does not enlarge independent errors).
  LayerNorm   (mer_layernorm_f16 / _ld_f16, two passes) the mean's sum rounds by (D / 256 + 13) u sum |x| (a chain of
              D / 256 pairwise-added values per thread, then the same 13 adds), moving every centred value by that
              / D; centring rounds u |x - mean|; the squares' sum (D / 256 + 13) u relative, r half of it + 3 u; the
              fma 2 u: own |gamma| / sigma (D / 256 + 13) u mean |x| + ((D / 256 + 13) / 2 + 5) u |gamma zhat| + u |y|.
              Carried: |gamma| / sigma times the error.
  linear      _lin_err with fp16 operands (u_op = 0: fp16-exact weights and activations, exact products), K the inner
              dimension; the epilogue's bias add rounds u |acc + b|, the residual add u |x|.
  RoPE        (x1 c - x2 s, x2 c + x1 s) in fp32 from fp16 q | k: two products and a sum, 2 u (|x1 c| + |x2 s|), rounded
              once to fp16.  Carried: |c| e1 + |s| e2 (the rotation of the q / k errors).
  attention   attention_tc_bound (the kernel's own error, with the fp16 ctx store) on the float64 q | k | v, plus the
              carried q / k / v errors: a v error reaches ctx through P in quadrature, sqrt(P^2 ev^2); a score error
              ds_ij = scale sqrt(eq_i^2 . k_j^2 + q_i^2 . ek_j^2) (quadrature over the head's columns) moves ctx by
              sum_j P_ij (ds_ij - sum_l P_il ds_il) v_j, at most 2 max_j ds_ij P |V|, the maximum over the keys row i
              sees.  Causal rows, ALiBi (an exact bias: its fp32 rounding is in attention_tc_bound's amplitude), the
              multi-query head (k / v errors of the one head shared by every query head) and head_dim 64 / 96 / 128.
  SwiGLU      h = a / (1 + expf(-a)) b: expf 2 ulp (relative 2 u of e^-a, <= 2 u of 1 + e^-a), the add, the division
              and the product: own 6 u |h|.  Carried: |silu'(a) b| ea + |silu(a)| eb + 1.1 ea eb + 0.25 |b| ea^2
              (|silu'| <= 1.1, |silu''| <= 0.5).
  tanh-GELU   gemm.cu gelu_tanh: x - x r or x r with r = t / (1 + t), t = 2^(-2.885 |v|), v = 0.79788456 x (1 +
              0.044715 x^2).  v's four roundings and the exponent's product give the exponent 6 u relative, i.e. t
              relative 2 |v| 6 u ln 2 ... <= 12 u |v|; ex2.approx 4 u, rcp.approx 2 u, 1 + t and r t 2 u: the small term
              x r is off by (8 + 12 |v|) u relative, and the final fma or product adds u |g|.  Carried: |g'| e + 0.4 e^2
              (|g''| <= 0.8).
  erf-GELU    _gelu_err (gelu_erf_fast, the MER_EPI_GELU epilogue).
  ReLU        relu(acc + b): slope <= 1, nothing of its own.
  stores      every value the CUDA path stores as fp16 (norm outputs, q | k | v, q | k after RoPE, the FFN activation)
              adds LAMBDA out_rounding (as _store in stack_layer); ctx's store is in attention_tc_bound.
"""
import math
import re

import numpy as np
import torch
import torch.nn.functional as F

import _kernel_refs as R

U = R.U32
FAMILIES = ("llama", "bloom", "opt", "gpt2", "falcon")
OPT_POS_OFFSET = 2

# Restated wiring faults (tests/test_decoder_refs.py: each leaves the bound by 4x or more on some element of a case the
# GPU test runs, in the families where it can act):
#   rope_pack_start   RoPE positions counted from the start of the packed batch instead of each sentence's
#   rope_off_by_one   RoPE at position p + 1
#                     Both shift every position of a sentence by one constant, and rotary scores depend on i - j only,
#                     so inside the table they change nothing but fp16 roundings.  They show where a position leaves
#                     the table: the rope kernel writes NaN there.  Hence the sentence of exactly max_position_embeddings
#                     tokens (its last row moves past the table) and a packed batch longer than the table (LLaMA)
#   rope_interleaved  RoPE on adjacent pairs (2 i, 2 i + 1) instead of rotate-half (i, i + head_dim / 2)
#   k_not_rotated     the rotation applied to q only
#   falcon_k_head     Falcon's rotation over `heads` heads instead of heads + 1: the one k head left unrotated
#   bloom_interleaved BLOOM's fused query_key_value rows read as q | k | v blocks (deinterleave_qkv skipped)
#   alibi_reversed    the ALiBi slopes in reversed head order
#   opt_offset0       OPT's learned positions read at p instead of p + 2 (hidden_states[0])
#   gpt2_no_types     GPT-2's wte[token_type] dropped (hidden_states[0])
#   swiglu_swap       SwiGLU's gate and up halves swapped: silu(up) gate
#   rms_as_ln         RMSNorm replaced by a LayerNorm (mean subtracted) with the same gain
#   falcon_sequential Falcon's MLP fed LN(x + attn) instead of the one LN(x) both branches share
#   drop_b_qkv, drop_b_o, drop_b_up, drop_b_down  a dropped bias of each biased GEMM (BLOOM, OPT, GPT-2)
#   no_residual       the attention half's output without the residual stream
# Not faults: ALiBi as slope * j versus slope * (j - i), or with j counted from the pack start (a per-row constant,
# which the softmax cancels).
DECODER_FAULTS = {
    "rope_pack_start": ("llama", "falcon"), "rope_off_by_one": ("llama", "falcon"),
    "rope_interleaved": ("llama", "falcon"), "k_not_rotated": ("llama",), "falcon_k_head": ("falcon",),
    "bloom_interleaved": ("bloom",), "alibi_reversed": ("bloom",), "opt_offset0": ("opt",),
    "gpt2_no_types": ("gpt2_types",), "swiglu_swap": ("llama",), "rms_as_ln": ("llama",),
    "falcon_sequential": ("falcon",), "drop_b_qkv": ("bloom", "opt", "gpt2"), "drop_b_o": ("bloom", "opt", "gpt2"),
    "drop_b_up": ("bloom", "opt", "gpt2"), "drop_b_down": ("bloom", "opt", "gpt2"), "no_residual": FAMILIES,
}
EMBED_FAULTS = ("opt_offset0", "gpt2_no_types")

# The packed batch of every small-checkpoint case: each kernel boundary +- 1 (16-key steps, 64-key tiles), an odd length
# first so that most sentence starts are not multiples of 8, and one of a few hundred; LLaMA, OPT and GPT-2 add one of
# exactly max_position_embeddings tokens (DECODER_MAX_POS), which reaches the last rotary row / learned position.
DECODER_LENS = [1, 2, 7, 8, 9, 63, 64, 65, 127, 128, 129, 300]
DECODER_MAX_POS = 320


def _small_cases():
    from mertools_b200 import synthetic as S
    long = DECODER_LENS + [DECODER_MAX_POS]
    return {
        # name: (family, state dict, heads, eps, max_pos, lens, token types)
        "llama": ("llama", lambda: S.llama_state_dict(seed=21, layers=4), 4, 1e-6, DECODER_MAX_POS, long, False),
        "bloom": ("bloom", lambda: S.bloom_state_dict(seed=23, layers=4), 4, 1e-5, None, DECODER_LENS, False),
        "opt": ("opt", lambda: S.opt_state_dict(seed=25, layers=4, max_pos=DECODER_MAX_POS), 4, 1e-5, DECODER_MAX_POS,
                long, False),
        "gpt2": ("gpt2", lambda: S.gpt2_state_dict(seed=29, layers=4, max_pos=DECODER_MAX_POS), 4, 1e-5,
                 DECODER_MAX_POS, long, False),
        "gpt2_types": ("gpt2", lambda: S.gpt2_state_dict(seed=29, layers=4, max_pos=DECODER_MAX_POS), 4, 1e-5,
                       DECODER_MAX_POS, long, True),
        "gpt2_96": ("gpt2", lambda: S.gpt2_state_dict(seed=31, vocab=4000, hidden=768, ffn=3072, layers=3,
                                                      max_pos=DECODER_MAX_POS), 8, 1e-5, DECODER_MAX_POS, long, False),
        "falcon": ("falcon", lambda: S.falcon_state_dict(seed=43, layers=4), 7, 1e-5, 2048, DECODER_LENS, False),
    }


def small_case(name):
    """dict(family, sd, heads, eps, max_pos, lens, ids, token_types, layers, vocab) of a small synthetic checkpoint case
    (the packed batch of DECODER_LENS; ids 0 and vocab - 1 both present, token types in 0 .. 2)."""
    family, make, heads, eps, max_pos, lens, types = _small_cases()[name]
    sd = make()
    emb = {"llama": "embed_tokens.weight", "bloom": "word_embeddings.weight", "opt": "decoder.embed_tokens.weight",
           "gpt2": "wte.weight", "falcon": "word_embeddings.weight"}[family]
    vocab = sd[emb].shape[0]
    rng = np.random.default_rng(7)
    ids = rng.integers(1, vocab - 1, sum(lens))
    ids[0], ids[-1] = 0, vocab - 1
    tt = rng.integers(0, 3, sum(lens)) if types else None
    layers = 1 + max(int(m.group(1)) for m in (re.match(r"(?:decoder\.)?(?:layers|h)\.(\d+)\.", k) for k in sd) if m)
    return dict(name=name, family=family, sd=sd, heads=heads, eps=eps, max_pos=max_pos, lens=list(lens), ids=ids,
                token_types=tt, layers=layers, vocab=vocab)


SMALL_CASES = ("llama", "bloom", "opt", "gpt2", "gpt2_types", "gpt2_96", "falcon")


def attention_kernel(family, hd):
    """The attention kernel instance a family's layer launches (attention_causal.cu)."""
    if family == "falcon":
        return "causal_attention_kernel<64, false, true>"
    return f"causal_attention_kernel<{hd}, {'true' if family == 'bloom' else 'false'}, false>"


# ---- weights ---------------------------------------------------------------------------------------------------------
def _get(sd, name, device):
    for k in (name, "decoder." + name, "transformer." + name, "model." + name):
        if k in sd:
            t = sd[k]
            t = torch.from_numpy(np.asarray(t)) if not torch.is_tensor(t) else t
            return t.to(device).half().double()
    raise KeyError(name)


def decoder_weights(family, sd, l, heads, device="cpu"):
    """Layer l of an HF-named state dict as float64 [out, in] matrices and vectors (fp16-rounded): ln1_g / ln1_b,
    wq / wk / wv and bq / bk / bv, wo / bo, ln2_g / ln2_b, w_up / b_up (w_gate for LLaMA), w_down / b_down; None where the
    family has no such parameter.  For the bloom_interleaved fault the raw fused rows come back too (qkv_raw, bqkv_raw)."""
    g = lambda n: _get(sd, n, device)  # noqa: E731
    w = dict.fromkeys(("ln1_b", "bq", "bk", "bv", "bo", "ln2_g", "ln2_b", "b_up", "b_down", "w_gate"))
    if family == "llama":
        p = f"layers.{l}."
        w.update(ln1_g=g(p + "input_layernorm.weight"), ln2_g=g(p + "post_attention_layernorm.weight"),
                 wq=g(p + "self_attn.q_proj.weight"), wk=g(p + "self_attn.k_proj.weight"),
                 wv=g(p + "self_attn.v_proj.weight"), wo=g(p + "self_attn.o_proj.weight"),
                 w_gate=g(p + "mlp.gate_proj.weight"), w_up=g(p + "mlp.up_proj.weight"),
                 w_down=g(p + "mlp.down_proj.weight"))
    elif family == "bloom":
        p = f"h.{l}."
        qkv, b = g(p + "self_attention.query_key_value.weight"), g(p + "self_attention.query_key_value.bias")
        D = qkv.shape[1]
        hd = D // heads
        wv3, bv3 = qkv.view(heads, 3, hd, D), b.view(heads, 3, hd)          # BloomAttention._split_heads
        w.update(qkv_raw=qkv, bqkv_raw=b,
                 wq=wv3[:, 0].reshape(D, D), wk=wv3[:, 1].reshape(D, D), wv=wv3[:, 2].reshape(D, D),
                 bq=bv3[:, 0].reshape(D), bk=bv3[:, 1].reshape(D), bv=bv3[:, 2].reshape(D))
        w.update(ln1_g=g(p + "input_layernorm.weight"), ln1_b=g(p + "input_layernorm.bias"),
                 wo=g(p + "self_attention.dense.weight"), bo=g(p + "self_attention.dense.bias"),
                 ln2_g=g(p + "post_attention_layernorm.weight"), ln2_b=g(p + "post_attention_layernorm.bias"),
                 w_up=g(p + "mlp.dense_h_to_4h.weight"), b_up=g(p + "mlp.dense_h_to_4h.bias"),
                 w_down=g(p + "mlp.dense_4h_to_h.weight"), b_down=g(p + "mlp.dense_4h_to_h.bias"))
    elif family == "opt":
        p = f"layers.{l}."
        a = p + "self_attn."
        w.update(ln1_g=g(p + "self_attn_layer_norm.weight"), ln1_b=g(p + "self_attn_layer_norm.bias"),
                 wq=g(a + "q_proj.weight"), wk=g(a + "k_proj.weight"), wv=g(a + "v_proj.weight"),
                 bq=g(a + "q_proj.bias"), bk=g(a + "k_proj.bias"), bv=g(a + "v_proj.bias"),
                 wo=g(a + "out_proj.weight"), bo=g(a + "out_proj.bias"),
                 ln2_g=g(p + "final_layer_norm.weight"), ln2_b=g(p + "final_layer_norm.bias"),
                 w_up=g(p + "fc1.weight"), b_up=g(p + "fc1.bias"), w_down=g(p + "fc2.weight"), b_down=g(p + "fc2.bias"))
    elif family == "gpt2":
        p = f"h.{l}."
        ca, cb = g(p + "attn.c_attn.weight"), g(p + "attn.c_attn.bias")        # Conv1D: [in, out], y @ W + b
        D = ca.shape[0]
        w.update(ln1_g=g(p + "ln_1.weight"), ln1_b=g(p + "ln_1.bias"),
                 wq=ca[:, :D].T, wk=ca[:, D:2 * D].T, wv=ca[:, 2 * D:].T, bq=cb[:D], bk=cb[D:2 * D], bv=cb[2 * D:],
                 wo=g(p + "attn.c_proj.weight").T, bo=g(p + "attn.c_proj.bias"),
                 ln2_g=g(p + "ln_2.weight"), ln2_b=g(p + "ln_2.bias"),
                 w_up=g(p + "mlp.c_fc.weight").T, b_up=g(p + "mlp.c_fc.bias"),
                 w_down=g(p + "mlp.c_proj.weight").T, b_down=g(p + "mlp.c_proj.bias"))
    else:
        p = f"h.{l}."
        qkv = g(p + "self_attention.query_key_value.weight")                   # heads x q | k | v, head_dim 64
        D = qkv.shape[1]
        hd = D // heads
        w.update(ln1_g=g(p + "input_layernorm.weight"), ln1_b=g(p + "input_layernorm.bias"),
                 wq=qkv[:heads * hd], wk=qkv[heads * hd:(heads + 1) * hd], wv=qkv[(heads + 1) * hd:],
                 wo=g(p + "self_attention.dense.weight"), w_up=g(p + "mlp.dense_h_to_4h.weight"),
                 w_down=g(p + "mlp.dense_4h_to_h.weight"))
    return w


# ---- stages ----------------------------------------------------------------------------------------------------------
def rms_err(x, e, w, eps):
    """(w x / rms(x), bound): carried |w| / rms e plus mer_rmsnorm's own (D / 512 + 12) u |y|."""
    D = x.shape[-1]
    rms = torch.sqrt((x * x).mean(-1, keepdim=True) + eps)
    y = w * (x / rms)
    return y, w.abs() / rms * e + (D / 512 + 12) * U * y.abs()


def ln_err(x, e, g, b, eps):
    """(LayerNorm(x), bound) of mer_layernorm_f16 / _ld_f16 (see the module docstring)."""
    D = x.shape[-1]
    mu = x.mean(-1, keepdim=True)
    sig = torch.sqrt(((x - mu) ** 2).mean(-1, keepdim=True) + eps)
    zg = (x - mu) / sig * g
    y = zg + b
    k = D / 256 + 13
    own = g.abs() / sig * k * U * x.abs().mean(-1, keepdim=True) + (k / 2 + 5) * U * zg.abs() + U * y.abs()
    return y, g.abs() / sig * e + own


def _lin(a, ea, wt, b, res=None, eres=None):
    """a @ wt.T (+ b) (+ res) with the GEMM's bound."""
    acc = a @ wt.T
    if b is not None:
        acc = acc + b
    z = acc if res is None else acc + res
    e = R._lin_err(lambda t, ww: t @ ww.T, a, ea, wt, 0.0, a.shape[-1])
    if b is not None:
        e = e + U * acc.abs()
    if res is not None:
        e = e + U * z.abs() + eres
    return z, e


def _store16(v, e):
    return v, e + R.LAMBDA * R.out_rounding(v, True)


def positions(lens, device, fault=None):
    pos = torch.cat([torch.arange(n) for n in lens]).to(device)
    if fault == "rope_pack_start":
        pos = torch.arange(sum(lens), device=device)
    if fault == "rope_off_by_one":
        pos = pos + 1
    return pos


def rope(x, e, cos, sin, pos, hd, interleaved=False):
    """Rotate-half rotary embedding of x [T, n heads x hd] at rows pos of the fp32 tables [max_pos, hd / 2]; returns
    (value, bound before the fp16 store).  A position past the table gives NaN, as the rope kernel writes there.
    interleaved: the adjacent-pair form (a fault)."""
    T = x.shape[0]
    inside = (pos < cos.shape[0])[:, None]
    nan = torch.tensor(float("nan"), dtype=torch.float64, device=x.device)
    c = torch.where(inside, cos.double()[pos.clamp(max=cos.shape[0] - 1)], nan)[:, None]
    s = torch.where(inside, sin.double()[pos.clamp(max=cos.shape[0] - 1)], nan)[:, None]
    xv, ev = x.reshape(T, -1, hd), e.reshape(T, -1, hd)
    if interleaved:
        x1, x2, e1, e2 = xv[..., 0::2], xv[..., 1::2], ev[..., 0::2], ev[..., 1::2]
    else:
        x1, x2, e1, e2 = xv[..., :hd // 2], xv[..., hd // 2:], ev[..., :hd // 2], ev[..., hd // 2:]
    a, b = x1 * c - x2 * s, x2 * c + x1 * s
    own = 2 * U * (x1 * c).abs() + 2 * U * (x2 * s).abs()
    own2 = 2 * U * (x2 * c).abs() + 2 * U * (x1 * s).abs()
    ea = c.abs() * e1 + s.abs() * e2 + own
    eb = c.abs() * e2 + s.abs() * e1 + own2
    if interleaved:
        out, eout = torch.stack([a, b], -1).reshape(T, -1), torch.stack([ea, eb], -1).reshape(T, -1)
    else:
        out, eout = torch.cat([a, b], -1).reshape(T, -1), torch.cat([ea, eb], -1).reshape(T, -1)
    return out, eout


def _rope_f32(x, cos, sin, pos, hd):
    """The rope kernel's arithmetic on fp32 values: products and the sum in fp32 (before the fp16 store)."""
    T = x.shape[0]
    c, s = cos.float()[pos][:, None], sin.float()[pos][:, None]
    xv = x.reshape(T, -1, hd)
    x1, x2 = xv[..., :hd // 2], xv[..., hd // 2:]
    return torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], -1).reshape(T, -1)


def attention_err(q, k, v, eq, ek, ev, lens, heads, hd, scale, slopes=None):
    """(ctx, bound) of the causal attention on float64 q [T, heads hd], k / v [T, kh hd] (kh = heads, or 1: multi-query)
    with bounds eq / ek / ev.  The bound is attention_tc_bound plus the carried errors (module docstring)."""
    mqa = k.shape[1] != q.shape[1]
    kh = 1 if mqa else heads
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    sl = None if slopes is None else slopes.to(q.device)
    ref, mag, amp, st = R.attention_packed(torch.cat([q, k] if mqa else [q, k, v], 1), cu, heads, hd, scale,
                                           causal=True, slopes=sl, v=v, mqa=mqa, stats=True)
    bound = R.attention_tc_bound(mag, amp, st, ref, "f16")
    D = heads * hd
    for s in range(len(lens)):
        a, b = cu[s], cu[s + 1]
        n = b - a
        hv = lambda t, h: t[a:b].reshape(n, h, hd).transpose(0, 1)  # noqa: E731
        qq, kk, vv, eqq, ekk, evv = hv(q, heads), hv(k, kh), hv(v, kh), hv(eq, heads), hv(ek, kh), hv(ev, kh)
        sc = qq @ kk.transpose(1, 2) * scale
        ii = torch.arange(n, device=q.device)
        if sl is not None:
            sc = sc + sl.double()[:, None, None] * ii[None, None, :]
        future = ii[None, :] > ii[:, None]
        p = torch.softmax(sc.masked_fill(future, float("-inf")), dim=-1)
        ds = torch.sqrt((eqq * eqq) @ (kk * kk).transpose(1, 2) + (qq * qq) @ (ekk * ekk).transpose(1, 2)) * scale
        ds = ds.masked_fill(future, 0.0)
        carried = torch.sqrt((p * p) @ (evv * evv)) + 2 * ds.amax(-1, keepdim=True) * (p @ vv.abs())
        bound[a:b] += carried.transpose(0, 1).reshape(n, D)
        del sc, p, ds, carried
    return ref, bound


def swiglu_err(a, b, ea, eb):
    s = torch.sigmoid(a)
    si = a * s
    h = si * b
    slope = (s * (1 + a * (1 - s))).abs()
    e = slope * b.abs() * ea + si.abs() * eb + 1.1 * ea * eb + 0.25 * b.abs() * ea * ea + 6 * U * h.abs()
    return h, e


GELU_C = 0.79788456


def gelu_tanh(x):
    return x * 0.5 * (1.0 + torch.tanh(GELU_C * x * (1 + 0.044715 * x * x)))


def gelu_tanh_err(z, e):
    v = GELU_C * z * (1 + 0.044715 * z * z)
    th = torch.tanh(v)
    g = 0.5 * z * (1 + th)
    slope = (0.5 * (1 + th) + 0.5 * z * (1 - th * th) * GELU_C * (1 + 3 * 0.044715 * z * z)).abs()
    t = torch.exp(-2 * v.abs())
    r = t / (1 + t)
    own = U * ((z * r).abs() * (8 + 12 * v.abs()) + g.abs())
    return g, slope * e + 0.4 * e * e + own


# ---- one layer -------------------------------------------------------------------------------------------------------
def _family_form(family, D, heads):
    hd = 64 if family == "falcon" else D // heads
    act = {"bloom": "gelu_tanh", "gpt2": "gelu_tanh", "opt": "relu", "falcon": "gelu", "llama": "swiglu"}[family]
    return hd, act


def decoder_layer(family, w, x_in, lens, heads, eps, tables=None, slopes=None, emulate=False, fault=None):
    """One decoder layer of `family` on x_in [tokens, hidden] (the GPU's hidden state l; Falcon's pad columns cut off)
    with packed sentence lengths `lens`, weights w (decoder_weights), rotary tables (cos, sin) (LLaMA, Falcon: rope_tables'
    fp32 values) or ALiBi slopes (BLOOM).  Returns (x_out, bound) in float64, or with `emulate` an fp32 evaluation that
    rounds every stored operand as the CUDA path does (bound None).  `fault` (DECODER_FAULTS) restates a wrong layer."""
    dt = torch.float32 if emulate else torch.float64
    x = x_in.to(dt)
    T, D = x.shape
    hd, act = _family_form(family, D, heads)
    W = {k: (None if v is None else v.to(dt)) for k, v in w.items()}
    dropped = {"drop_b_qkv": ("bq", "bk", "bv"), "drop_b_o": ("bo",), "drop_b_up": ("b_up",),
               "drop_b_down": ("b_down",)}.get(fault, ())
    for name in dropped:
        if W[name] is not None:
            W[name] = torch.zeros_like(W[name])
    if fault == "bloom_interleaved":
        W["wq"], W["wk"], W["wv"] = W["qkv_raw"][:D], W["qkv_raw"][D:2 * D], W["qkv_raw"][2 * D:]
        W["bq"], W["bk"], W["bv"] = W["bqkv_raw"][:D], W["bqkv_raw"][D:2 * D], W["bqkv_raw"][2 * D:]
    zero = torch.zeros_like(x)
    f16 = lambda v: R.f16_satfinite(v)  # noqa: E731

    def norm(v, ev, g, b):
        if family == "llama" and fault != "rms_as_ln":
            if emulate:
                return f16(g * (v * torch.rsqrt(v.pow(2).mean(-1, keepdim=True) + eps))), None
            return _store16(*rms_err(v, ev, g, eps))
        if emulate:
            return f16(F.layer_norm(v, (D,), g, b, eps)), None
        return _store16(*ln_err(v, ev, g, torch.zeros_like(g) if b is None else b, eps))

    def lin(a, ea, wn, bn, res=None, eres=None):
        if emulate:
            z = a @ W[wn].T
            z = z if W[bn] is None else z + W[bn]
            return (z if res is None else z + res), None
        return _lin(a, ea, W[wn], W[bn], res, eres)

    # attention half
    y, ey = norm(x, zero, W["ln1_g"], W["ln1_b"])
    q, eq = lin(y, ey, "wq", "bq")
    k, ek = lin(y, ey, "wk", "bk")
    v, ev = lin(y, ey, "wv", "bv")
    if emulate:
        q, k, v = f16(q), f16(k), f16(v)
    else:
        (q, eq), (k, ek), (v, ev) = _store16(q, eq), _store16(k, ek), _store16(v, ev)
    if tables is not None:
        pos = positions(lens, x.device, fault)
        cos, sin = tables
        inter = fault == "rope_interleaved"
        rot_k = fault not in ("k_not_rotated", "falcon_k_head")
        if emulate:
            q = f16(_rope_f32(q, cos, sin, pos, hd))
            k = f16(_rope_f32(k, cos, sin, pos, hd)) if rot_k else k
        else:
            q, eq = _store16(*rope(q, eq, cos, sin, pos, hd, inter))
            if rot_k:
                k, ek = _store16(*rope(k, ek, cos, sin, pos, hd, inter))
    sl = slopes
    if sl is not None and fault == "alibi_reversed":
        sl = sl.flip(0)
    scale = hd ** -0.5
    if emulate:
        cu = [0]
        for n in lens:
            cu.append(cu[-1] + n)
        mqa = family == "falcon"
        ctx = R.attention_tc_emulated(torch.cat([q, k] if mqa else [q, k, v], 1), cu, heads, hd,
                                      float(np.float32(scale)), causal=True, slopes=sl, v=v, mqa=mqa)
        ctx, ectx = f16(ctx), None
    else:
        ctx, ectx = attention_err(q, k, v, eq, ek, ev, lens, heads, hd, scale, sl)
    res = None if fault == "no_residual" else x
    eres = None if emulate else zero
    if family == "falcon":                    # x + dense(ctx) + dense_4h_to_h(gelu(dense_h_to_4h(y)))
        x1, ex1 = lin(ctx, ectx, "wo", "bo", res, eres)
        y2, ey2 = (y, ey) if fault != "falcon_sequential" else norm(x1, ex1, W["ln1_g"], W["ln1_b"])
        z, ez = lin(y2, ey2, "w_up", "b_up")
        if emulate:
            h = f16(0.5 * z * (1 + torch.erf(z / math.sqrt(2.0))))
            return x1 + h @ W["w_down"].T, None
        h, eh = _store16(*R._gelu_err(z, ez))
        return lin(h, eh, "w_down", "b_down", x1, ex1)
    x1, ex1 = lin(ctx, ectx, "wo", "bo", res, eres)
    y2, ey2 = norm(x1, ex1, W["ln2_g"], W["ln2_b"])
    if family == "llama":
        gate, up = ("w_up", "w_gate") if fault == "swiglu_swap" else ("w_gate", "w_up")
        a, ea = lin(y2, ey2, gate, "b_up")
        b, eb = lin(y2, ey2, up, "b_up")
        if emulate:
            h = f16(a / (1.0 + torch.exp(-a)) * b)
        else:
            h, eh = _store16(*swiglu_err(a, b, ea, eb))
    else:
        z, ez = lin(y2, ey2, "w_up", "b_up")
        if emulate:
            h = f16(torch.relu(z) if act == "relu" else gelu_tanh(z))
        elif act == "relu":
            h, eh = _store16(torch.relu(z), ez)
        else:
            h, eh = _store16(*gelu_tanh_err(z, ez))
    return lin(h, None if emulate else eh, "w_down", "b_down", x1, None if emulate else ex1)


# ---- hidden_states[0] and the final norm -----------------------------------------------------------------------------
def decoder_embedding(family, sd, ids, lens, eps=None, token_types=None, fault=None, device="cpu"):
    """(hidden_states[0], bound) of a family on packed ids: LLaMA / Falcon E[ids] (exact: bound 0); BLOOM
    word_embeddings_layernorm(E[ids]) stored fp32; OPT E[ids] + P[p + 2] (one fp32 add); GPT-2 wte[ids] + wpe[p]
    (+ wte[token_types]) (one or two fp32 adds).  p counts from each sentence's start."""
    ids = torch.as_tensor(np.asarray(ids), device=device)
    pos = positions(lens, device)
    if family in ("llama", "falcon"):
        E = _get(sd, "embed_tokens.weight" if family == "llama" else "word_embeddings.weight", device)
        x = E[ids]
        return x, torch.zeros_like(x)
    if family == "bloom":
        x = _get(sd, "word_embeddings.weight", device)[ids]
        return ln_err(x, torch.zeros_like(x), _get(sd, "word_embeddings_layernorm.weight", device),
                      _get(sd, "word_embeddings_layernorm.bias", device), eps)
    if family == "opt":
        a = _get(sd, "embed_tokens.weight", device)[ids]
        x = a + _get(sd, "embed_positions.weight", device)[pos + (0 if fault == "opt_offset0" else OPT_POS_OFFSET)]
        return x, U * x.abs()
    E = _get(sd, "wte.weight", device)
    x = E[ids] + _get(sd, "wpe.weight", device)[pos]
    e = U * x.abs()
    if token_types is not None and fault != "gpt2_no_types":
        x = x + E[torch.as_tensor(np.asarray(token_types), device=device)]
        e = e + U * x.abs()
    return x, e


def final_norm(family, sd, x, e, eps, device="cpu"):
    """(hidden_states[L], bound): the final norm (LLaMA norm, BLOOM / GPT-2 / Falcon ln_f, OPT final_layer_norm) of the
    last layer's output, stored fp32."""
    if family == "llama":
        return rms_err(x, e, _get(sd, "norm.weight", device), eps)
    name = "final_layer_norm" if family == "opt" else "ln_f"
    return ln_err(x, e, _get(sd, name + ".weight", device), _get(sd, name + ".bias", device), eps)


def layer_tables(family, max_pos, theta=10000.0, heads=None, device="cpu"):
    """(tables, slopes) decoder_layer takes for a family: rope_tables' fp32 cos / sin (LLaMA at head_dim 128, Falcon at
    64), alibi_slopes (BLOOM)."""
    from mertools_b200.extract.ln_decoder_text import alibi_slopes
    from mertools_b200.extract.llama_text import rope_tables
    if family == "llama":
        return tuple(t.to(device) for t in rope_tables(max_pos, theta)), None
    if family == "falcon":
        return tuple(t.to(device) for t in rope_tables(max_pos, theta, 64)), None
    if family == "bloom":
        return None, alibi_slopes(heads).to(device)
    return None, None
