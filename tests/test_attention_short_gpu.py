"""GPU parity of the short-sequence fp16 attention kernel (attention_short.cu: one CTA per (sequence, head), rows of
<= 249 tokens) against a float64 softmax(Q K^T / 8) V of the same fp16 operand values, in every ctx format, and
against the 64 x 64-tile kernel of attention_f16.cu (MER_ATT_SHORT=0).  MER_ATT_SHORT=1 sends every batch of the
module to the short kernel (by default it takes batches whose longest row has 129 .. 208 tokens)."""
import os

import pytest
import torch

from mertools_b200 import _lib as L

pytestmark = pytest.mark.gpu
HD = 64
# every 16-key step boundary the kernel has (1 / 2 chunks, partial steps, the 128-key chunk edge, the 249 maximum
# whose keys fill all 256 key positions when its start is not a multiple of 8),
# in an order that makes most starts not multiples of 8
LENS = [1, 2, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64, 65, 127, 128, 129, 196, 197, 198, 208, 240, 241, 247, 248,
        249, 249]


def _ragged(lens):
    # interleave odd lengths so that starts are mostly not multiples of 8
    return [lens[i] for i in range(len(lens)) if i % 2 == 0] + [lens[i] for i in range(len(lens)) if i % 2 == 1]


def _reference(q, k, v, cu, heads):
    out = torch.zeros(q.shape, dtype=torch.float64)
    for s in range(len(cu) - 1):
        a, b = cu[s], cu[s + 1]
        for h in range(heads):
            c = slice(h * HD, (h + 1) * HD)
            p = torch.softmax(q[a:b, c] @ k[a:b, c].T / 8.0, dim=-1)
            out[a:b, c] = p @ v[a:b, c]
    return out


def _operands(lens, heads, cuda, scale=1.5, nan_pad=False):
    g = torch.Generator().manual_seed(23)
    tokens = sum(lens)
    qkv = (torch.randn(tokens, 3 * heads * HD, generator=g) * scale).to(torch.float16)
    host = qkv.double()
    ref = None
    cu = [0]
    for n in lens:
        cu.append(cu[-1] + n)
    ref = _reference(host[:, :heads * HD], host[:, heads * HD:2 * heads * HD], host[:, 2 * heads * HD:], cu, heads)
    qkv = qkv.to(cuda)
    ld = (tokens + 7) // 8 * 8 + (64 if nan_pad else 0)
    vt = torch.full((heads * HD, ld), float("nan") if nan_pad else 0.0, dtype=torch.float16, device=cuda)
    vt[:, :tokens] = qkv[:, 2 * heads * HD:].T
    if nan_pad:
        qkv[:, 2 * heads * HD:] = float("nan")  # the V columns are never read: the QKV GEMM writes V^T instead
    return qkv, vt, torch.tensor(cu, dtype=torch.int32, device=cuda), ref


class _env:
    def __init__(self, name, value):
        self.name, self.value = name, value

    def __enter__(self):
        self.old = os.environ.get(self.name)
        os.environ[self.name] = str(self.value)

    def __exit__(self, *a):
        if self.old is None:
            os.environ.pop(self.name, None)
        else:
            os.environ[self.name] = self.old


def _run(qkv, vt, cu, lens, heads, dtype, short=1, **kw):
    ctx = torch.full((qkv.shape[0], heads * HD), float("nan"), dtype=dtype, device=qkv.device)
    with _env("MER_ATT_SHORT", short):
        L.attention(qkv, ctx, cu, max(lens), heads, vt=vt, **kw)
    torch.cuda.synchronize()
    return ctx


def _rel(out, ref):
    return float((out.double().cpu() - ref).abs().max() / ref.abs().max())


@pytest.mark.parametrize("heads", [3, 12])
def test_short_attention_f16_out_vs_float64(cuda, heads):
    lens = _ragged(LENS)
    qkv, vt, cu, ref = _operands(lens, heads, cuda)
    out = _run(qkv, vt, cu, lens, heads, torch.float16)
    assert torch.isfinite(out).all()
    err = _rel(out, ref)
    assert err < 2e-3, err  # fp16 P and the fp16 output rounding


@pytest.mark.parametrize("mode", ["fp32", "tf32", "split"])
def test_short_attention_fp32_ctx_formats(cuda, mode):
    lens = _ragged(LENS)
    qkv, vt, cu, ref = _operands(lens, 3, cuda)
    ctx = _run(qkv, vt, cu, lens, 3, torch.float32, round_out=(mode == "tf32"), split_out=(mode == "split"))
    out = L.unsplit_bf16(ctx) if mode == "split" else ctx
    assert torch.isfinite(out).all()
    err = _rel(out, ref)
    assert err < 1e-3, err  # fp16 P only
    if mode == "tf32":
        assert int((ctx.view(torch.int32) & 0x1FFF).abs().max()) == 0  # low 13 mantissa bits cleared


def test_short_attention_peaked_scores(cuda):
    """Operand scale 4: scores of +-60 before the 1/8 scale; the 2-chunk rows rescale once by a large factor."""
    lens = [197, 249, 3, 129, 248, 64]
    qkv, vt, cu, ref = _operands(lens, 3, cuda, scale=4.0)
    out = _run(qkv, vt, cu, lens, 3, torch.float32)
    assert torch.isfinite(out).all()
    err = _rel(out, ref)
    assert err < 1e-3, err


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_short_attention_ignores_padding(cuda, dtype):
    """NaN in the V^T columns past `tokens` and in the unused V columns of qkv: masked keys (P = 0) must meet the
    zero fill of the V^T load, never the padding."""
    lens = [5, 197, 249, 17, 131]  # the last sequence ends inside a 64-key V^T box
    qkv, vt, cu, ref = _operands(lens, 3, cuda, nan_pad=True)
    out = _run(qkv, vt, cu, lens, 3, dtype)
    assert torch.isfinite(out).all()
    assert _rel(out, ref) < (2e-3 if dtype == torch.float16 else 1e-3)


@pytest.mark.parametrize("heads", [3, 12])
def test_short_attention_agrees_with_tile_kernel(cuda, heads):
    """The same fp16 probabilities as the 64 x 64-tile kernel (MER_ATT_SHORT=0), another summation order."""
    lens = _ragged(LENS)
    qkv, vt, cu, ref = _operands(lens, heads, cuda)
    a = _run(qkv, vt, cu, lens, heads, torch.float16)
    b = _run(qkv, vt, cu, lens, heads, torch.float16, short=0)
    assert torch.isfinite(b).all()
    d = float((a.double() - b.double()).abs().max().cpu() / ref.abs().max())
    assert d < 1.5e-3, d


def test_vit_rows_take_the_short_kernel_by_default(cuda):
    """197-token rows (ViT-B/16) reach the short kernel without MER_ATT_SHORT: same result as forcing it."""
    lens = [197] * 6
    qkv, vt, cu, ref = _operands(lens, 12, cuda)
    old = os.environ.pop("MER_ATT_SHORT", None)
    try:
        ctx = torch.full((qkv.shape[0], 12 * HD), float("nan"), dtype=torch.float16, device=cuda)
        L.attention(qkv, ctx, cu, 197, 12, vt=vt)
        torch.cuda.synchronize()
    finally:
        if old is not None:
            os.environ["MER_ATT_SHORT"] = old
    forced = _run(qkv, vt, cu, lens, 12, torch.float16)
    assert torch.equal(ctx, forced)
    assert _rel(ctx, ref) < 2e-3
