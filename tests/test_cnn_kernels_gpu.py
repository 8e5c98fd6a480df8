"""Kernel-level parity of the convolutional extractors' kernels (resnet.cu) against float64 (tests/_kernel_refs.py).

Table-driven executor (mer_cnn_forward): each case is a four-part op table -- a STEM on a small frame, SHAPE ops that
declare the input maps of the op under test, the op, and a GAP -- run on a workspace prefilled with NaN into which the
test writes the declared inputs (nothing writes them during the call).  Outputs are read straight from the workspace:
its layout is mirrored by _kernel_refs.cnn_plan, whose total must equal mer_cnn_workspace_bytes.  Every case checks
  - the op against float64 computed on the operand values, element by element: GEMM-backed ops (STEM, CONV) normalised
    by |x| |w| + |b| + |res| at the GEMM tests' bar of 2^-16; max-pool, crop, slice, upsample-add bit for bit (one fp32
    add rounds like the float64 sum rounded to fp32); affine, mask-multiply, GAP, SE and CBAM under fp32 bounds
    written out from their reduction lengths;
  - that no NaN is left where the op writes;
  - that frames 1.. of the output are bit-identical when frame 0's input holds NaN or 1e30;
  - that a stored-but-not-real channel range (C < Cs) comes out as the op promises.
Max-pool is never fed NaN for the comparison with torch: fmaxf drops a NaN operand where torch's max-pool propagates it.

Fixed graphs: the ResNet-18 stem output and pre-pool map, and the VGGish pool4 map and fc1_1 output, read from the
buffers mer_resnet18_forward / mer_vggish_forward leave behind (layouts mirrored from ResnetPlan / VggishPlan)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _kernel_refs as R
from mertools_b200 import _lib as L
from mertools_b200 import encoders as En

pytestmark = pytest.mark.gpu
F16, BF = L.MER_GEMM_F16, L.MER_GEMM_BF16X3
BAR = 2.0 ** -16
U = 2.0 ** -24
STEM, CONV, MAXPOOL, GAP, SE, CROP, SHAPE, SLICE, CBAM, AFFINE, UPADD, MASKMUL = range(12)
IN = 1  # buffer of the op's first input (declared by SHAPE)


def _lib():
    lib = L.lib()
    lib.mer_cnn_workspace_bytes.restype = C.c_longlong
    lib.mer_cnn_workspace_bytes.argtypes = [C.POINTER(En.MerCnnModel), C.c_int]
    fwd = L.declare("mer_cnn_forward", [C.POINTER(En.MerCnnModel), C.c_void_p, C.c_int, C.c_void_p, C.c_longlong,
                                        C.c_void_p, C.c_void_p])
    return lib, fwd


class Store:
    """Device copies of GEMM weights (fp16 or split bf16 per mode) and plain fp32 tables, by address -> fp32 values."""

    def __init__(self, dev, mode):
        self.dev, self.mode, self.vals, self.keep = dev, mode, {}, []

    def _put(self, host, dev_t):
        self.keep.append(dev_t)
        self.vals[dev_t.data_ptr()] = host
        return dev_t.data_ptr()

    def gemm(self, w, b):
        w = w.float()
        if self.mode == F16:
            w = R.f16_satfinite(w)
            wd = w.half().to(self.dev)
        else:
            wd = L.split_bf16(w.to(self.dev).contiguous())
        return self._put(w, wd), self._put(b.float(), b.float().to(self.dev))

    def dense(self, w, b):
        return self._put(w.float(), w.float().to(self.dev).contiguous()), self._put(b.float(), b.float().to(self.dev))


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _conv_entry(st, cin, cout, cout_pad, k, stride, pad, seed, kpad=None, junk_rows=False):
    kk = k * k * cin
    kpad = kk if kpad is None else kpad
    w = torch.zeros(cout_pad, kpad)
    w[:cout, :kk] = torch.randn(cout, kk, generator=_g(seed)) * math.sqrt(2.0 / kk)
    b = torch.zeros(cout_pad)
    b[:cout] = 0.1 * torch.randn(cout, generator=_g(seed + 1))
    if junk_rows:   # rows past cout: the GEMM computes them, an op reading only the real channels must ignore them
        w[cout:, :kk] = torch.randn(cout_pad - cout, kk, generator=_g(seed + 2))
        b[cout:] = 5.0
    wp, bp = st.gemm(w, b)
    return dict(w=wp, b=bp, cin=cin, cout=cout, cout_pad=cout_pad, k=k, stride=stride, pad=pad, kpad=kpad)


def _stem_entry(st, seed, cout=128, cout_pad=128):
    return _conv_entry(st, 3, cout, cout_pad, 7, 2, 3, seed, kpad=192 if st.mode == F16 else 160)


def _frames(n, h, w, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, h, w, 3), dtype=np.uint8)


def _run(cuda, m, frames, inputs, poison=None):
    """mer_cnn_forward on a NaN-filled workspace with `inputs` {buffer: [n, H, W, Cs] fp32} written into their buffers.
    Returns (out_feats, {buffer: [n, H, W, Cs] as left}) after checking the mirrored layout and the return code."""
    lib, fwd = _lib()
    n = len(frames)
    off, sh = R.cnn_plan(m, n)
    assert lib.mer_cnn_workspace_bytes(C.byref(m), n) == off["total"]
    ws = torch.full((off["total"] // 4,), float("nan"), device=cuda)

    def view(b):
        H, W, _, Cs = sh[b]
        return ws[off[b] // 4: off[b] // 4 + n * H * W * Cs].view(n, H, W, Cs)
    for b, t in inputs.items():
        assert tuple(t.shape[1:]) == (sh[b][0], sh[b][1], sh[b][3]), (b, t.shape, sh[b])
        view(b).copy_(t)
    out = torch.full((n, m.feat_dim), float("nan"), device=cuda)
    fr = torch.from_numpy(np.ascontiguousarray(frames)).to(cuda)
    before = L.launch_count()
    rc = fwd(C.byref(m), L.ptr(fr), n, L.ptr(ws), off["total"], L.ptr(out), L.stream_ptr())
    assert rc == 0, L.lib().mer_last_error()
    torch.cuda.synchronize()
    assert L.launch_count() > before
    return out.cpu(), {b: view(b).cpu() for b in sh}


def _table(st, hw, mid, convs, feat_src, feat_dim, inputs_cs, gap_p=(0, 0, 0)):
    """STEM on a (2 H - 1) x (2 W - 1) frame (output H x W into buffer 0), one SHAPE per entry of inputs_cs {buffer: Cs},
    the ops `mid`, a GAP of feat_src.  Conv entry 0 is the stem; `convs` follow from index 1."""
    ops = [dict(kind=STEM, conv=0, dst=0, relu=1)]
    ops += [dict(kind=SHAPE, src=0, dst=b, p=(cs,)) for b, cs in inputs_cs.items()]
    ops += mid + [dict(kind=GAP, src=feat_src, p=gap_p)]
    m, keep = R.cnn_model([_stem_entry(st, 900)] + convs, ops, st.mode, (2 * hw[0] - 1, 2 * hw[1] - 1), feat_dim,
                          scale=1 / 255, mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225))
    return m, keep


def _check_neighbours(cuda, m, frames, inputs, outs, poison):
    """Frame 0 of every input := poison; frames 1.. of buffers `outs` must match the clean run bit for bit."""
    _, clean = _run(cuda, m, frames, inputs)
    bad = {b: t.clone() for b, t in inputs.items()}
    for t in bad.values():
        t[0] = poison
    _, dirty = _run(cuda, m, frames, bad)
    for b in outs:
        assert torch.equal(R.bits(clean[b][1:]), R.bits(dirty[b][1:])), f"frame 0 ({poison}) leaked into buffer {b}"


def _ref(m, st, frames, inputs):
    return R.interpret_cnn_tables(m, st.vals, frames, dtype=torch.float64, bufs={b: t.cpu() for b, t in inputs.items()},
                                  operands=True)


# ---------------------------------------------------------------------------------------------------------------------
# STEM
@pytest.mark.parametrize("mode", [F16, BF])
@pytest.mark.parametrize("hw", [(224, 224), (33, 17), (1, 1)])
def test_stem_vs_float64(cuda, mode, hw):
    """The fused gather (BGR -> RGB, fma(pix, scale, -mean) / std, zero padding, fp16 or split operand) and the GEMM.
    Unequal mean, std and scale per channel: a channel swap moves every operand."""
    st = Store(cuda, mode)
    n = 3
    stem = _stem_entry(st, 11, cout=64, cout_pad=128)
    m, _keep = R.cnn_model([stem], [dict(kind=STEM, conv=0, dst=0, relu=1), dict(kind=GAP, src=0)], mode, hw, 64,
                           scale=1 / 255, mean=(0.61, 0.2, 0.33), std=(0.15, 0.4, 0.27))
    frames = _frames(n, hw[0], hw[1], 5)
    out, bufs = _run(cuda, m, frames, {})
    got = bufs[0].double()
    x = R.stem_operand(frames, m.scale, [m.mean[i] for i in range(3)], [m.std[i] for i in range(3)])
    y, a = R.cnn_conv(x, st.vals[stem["w"]], st.vals[stem["b"]], 7, 2, 3, mode)
    e = float(((got - torch.relu(y)).abs() / a.clamp(min=1e-30)).max())
    print(f"stem {'f16' if mode == F16 else 'split'} {hw}: normalised error {e:.2e}")
    assert e < BAR and not torch.isnan(got).any()
    assert bool((bufs[0][..., 64:] == 0).all()), "padded channels of the stem output"
    # a plain pix * scale - mean operand is off by an ulp in some of these pixels: the emulation is what is compared
    assert got.shape == (n, (hw[0] - 1) // 2 + 1, (hw[1] - 1) // 2 + 1, 128)
    hw_out = got.shape[1] * got.shape[2]
    gref = got[..., :64].mean(dim=(1, 2))
    assert bool(((out.double() - gref).abs() <= (hw_out + 3) * U * got[..., :64].abs().mean(dim=(1, 2)) + 1e-30).all())
    if hw == (33, 17):   # frame 0 changed: frames 1.. of the output unchanged
        fr2 = frames.copy()
        fr2[0] = 255 - fr2[0]
        _, b2 = _run(cuda, m, fr2, {})
        assert torch.equal(R.bits(b2[0][1:]), R.bits(bufs[0][1:])) and not torch.equal(b2[0][0], bufs[0][0])


# ---------------------------------------------------------------------------------------------------------------------
# CONV
CONV_CASES = [
    # (k, stride, pad, (H, W), cin, Cs, c0, cout, cout_pad, relu, res, n)     res: None / "distinct" / "inplace"
    (1, 1, 0, (7, 7), 64, 64, 0, 128, 128, 1, None, 3),
    (1, 2, 0, (13, 9), 64, 128, 64, 256, 256, 0, "distinct", 2),
    (3, 1, 1, (14, 14), 64, 128, 0, 64, 128, 1, None, 2),
    (3, 2, 1, (13, 9), 64, 192, 128, 128, 128, 1, "inplace", 3),
    (3, 1, 1, (1, 1), 128, 128, 0, 512, 512, 0, "distinct", 4),
    (3, 1, 1, (2, 3), 64, 64, 0, 128, 128, 1, "inplace", 2),
    (7, 2, 3, (14, 14), 64, 64, 0, 128, 128, 1, None, 2),
    (1, 1, 0, (14, 14), 128, 256, 64, 128, 128, 1, None, 97),     # 97 * 196 rows: 149 row tiles of 128 (> 132 CTAs)
    (3, 1, 1, (7, 7), 64, 64, 0, 64, 128, 0, "distinct", 5),      # 245 rows: one full and one ragged row tile
]


@pytest.mark.parametrize("mode", [F16, BF])
@pytest.mark.parametrize("case", range(len(CONV_CASES)))
def test_conv_vs_float64(cuda, mode, case):
    """im2col gather (fp16 / split operand) + GEMM with bias, residual (distinct or in place, res == dst) and ReLU."""
    k, s, pad, hw, cin, cs, c0, cout, cout_pad, relu, res, n = CONV_CASES[case]
    st = Store(cuda, mode)
    cv = _conv_entry(st, cin, cout, cout_pad, k, s, pad, 100 + case)
    oh, ow = (hw[0] + 2 * pad - k) // s + 1, (hw[1] + 2 * pad - k) // s + 1
    x = torch.randn(n, hw[0], hw[1], cs, generator=_g(case)) * 2
    x[..., :c0] = float("nan")                      # channels outside [c0, c0 + cin) are never read
    x[..., c0 + cin:] = float("nan")
    inputs_cs = {IN: cs}
    inputs = {IN: x.to(cuda)}
    dst, rb = 3, -1
    if res:
        rb = 2 if res == "distinct" else 3
        r = torch.randn(n, oh, ow, cout_pad, generator=_g(case + 50))
        r[..., cout:] = 0.0
        inputs_cs[rb] = cout_pad
        inputs[rb] = r.to(cuda)
    mid = [dict(kind=CONV, conv=1, src=IN, dst=dst, res=rb, relu=relu, p=(c0,))]
    if res and (oh, ow) != hw:      # declare the residual at the output size: SHAPE of a crop of the stem output
        mid = [dict(kind=CROP, src=0, dst=4, p=(0, 0, oh, ow)), dict(kind=SHAPE, src=4, dst=rb, p=(cout_pad,))] + mid
        inputs_cs.pop(rb)
    m, _keep = _table(st, hw, mid, [cv], dst, cout, inputs_cs)
    out, bufs = _run(cuda, m, _frames(n, 2 * hw[0] - 1, 2 * hw[1] - 1, 1), inputs)
    got = bufs[dst].double()
    y, a = R.cnn_conv(x[..., c0:c0 + cin], st.vals[cv["w"]], st.vals[cv["b"]], k, s, pad, mode,
                      res=None if rb < 0 else inputs[rb].cpu())
    if relu:
        y = torch.relu(y)
    e = float(((got - y).abs() / a.clamp(min=1e-30)).max())
    print(f"conv {CONV_CASES[case]} {'f16' if mode == F16 else 'split'}: normalised error {e:.2e}")
    assert got.shape == (n, oh, ow, cout_pad) and not torch.isnan(got).any()
    assert e < BAR
    if cout < cout_pad and rb < 0:
        assert bool((bufs[dst][..., cout:] == 0).all()), "padded output channels"
    if case in (1, 3, 8):
        _check_neighbours(cuda, m, _frames(n, 2 * hw[0] - 1, 2 * hw[1] - 1, 1), inputs, [dst], float("nan"))


# ---------------------------------------------------------------------------------------------------------------------
# MAXPOOL
POOL_SIZES = [(2, 3), (3, 4), (4, 5), (5, 6), (6, 7), (7, 2), (55, 56), (111, 112), (113, 113)]


@pytest.mark.parametrize("pad,ceil", [(1, 0), (0, 1)])
@pytest.mark.parametrize("hw", POOL_SIZES)
def test_maxpool3x3s2_is_torch_bit_for_bit(cuda, pad, ceil, hw):
    """MaxPool2d(3, 2, pad 1) (torchvision) and MaxPool2d(3, 2, 0, ceil_mode=True) (FER+) on all-negative maps, so
    that a window clipped at the bottom-right edge or padding read as 0 shows; output sizes are torch's."""
    st = Store(cuda, F16)
    n = 3
    x = -(torch.rand(n, hw[0], hw[1], 128, generator=_g(hw[0])) + 0.01)
    m, _keep = _table(st, hw, [dict(kind=MAXPOOL, src=IN, dst=2, k=3, stride=2, pad=pad, ceil_mode=ceil)], [], 2, 128,
                      {IN: 128})
    frames = _frames(n, 2 * hw[0] - 1, 2 * hw[1] - 1, 2)
    _, bufs = _run(cuda, m, frames, {IN: x.to(cuda)})
    want = F.max_pool2d(x.permute(0, 3, 1, 2), 3, 2, pad, ceil_mode=bool(ceil)).permute(0, 2, 3, 1)
    assert bufs[2].shape == want.shape and torch.equal(R.bits(bufs[2]), R.bits(want.contiguous()))
    if hw in ((5, 6), (111, 112)):
        _check_neighbours(cuda, m, frames, {IN: x.to(cuda)}, [2], 1e30)


@pytest.mark.parametrize("hw", [(2, 2), (96, 64), (14, 14)])
def test_maxpool2x2_is_torch_bit_for_bit(cuda, hw):
    st = Store(cuda, BF)
    n = 2
    x = -(torch.rand(n, hw[0], hw[1], 128, generator=_g(7)) + 0.01)
    m, _keep = _table(st, hw, [dict(kind=MAXPOOL, src=IN, dst=2, k=2, stride=2)], [], 2, 128, {IN: 128})
    frames = _frames(n, 2 * hw[0] - 1, 2 * hw[1] - 1, 2)
    _, bufs = _run(cuda, m, frames, {IN: x.to(cuda)})
    want = F.max_pool2d(x.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1).contiguous()
    assert torch.equal(R.bits(bufs[2]), R.bits(want))
    _check_neighbours(cuda, m, frames, {IN: x.to(cuda)}, [2], 1e30)


# ---------------------------------------------------------------------------------------------------------------------
# CROP, SLICE, UPADD, AFFINE, MASKMUL
@pytest.mark.parametrize("win", [(0, 0, 1, 1), (6, 8, 1, 1), (0, 0, 7, 9), (2, 0, 3, 9), (0, 3, 7, 2), (6, 0, 1, 9)])
def test_crop_bit_for_bit(cuda, win):
    st = Store(cuda, F16)
    n = 2
    x = torch.randn(n, 7, 9, 128, generator=_g(8))
    m, _keep = _table(st, (7, 9), [dict(kind=CROP, src=IN, dst=2, p=win)], [], 2, 128, {IN: 128})
    frames = _frames(n, 13, 17, 3)
    _, bufs = _run(cuda, m, frames, {IN: x.to(cuda)})
    y0, x0, h, w = win
    assert torch.equal(R.bits(bufs[2]), R.bits(x[:, y0:y0 + h, x0:x0 + w].contiguous()))
    _check_neighbours(cuda, m, frames, {IN: x.to(cuda)}, [2], float("nan"))


@pytest.mark.parametrize("relu", [0, 1, 2])
@pytest.mark.parametrize("form", ["plain", "addend", "inplace"])
@pytest.mark.parametrize("width", [4, 32])
def test_slice_bit_for_bit(cuda, relu, form, width):
    """dst[..., d0 : d0 + w] = f(src[..., s0 : s0 + w]) (+ res[..., r0 : r0 + w]); the rest of dst keeps what it held."""
    st = Store(cuda, F16)
    n = 2
    s0, d0, r0 = 8, 12, 20 if form != "inplace" else 12
    src = torch.randn(n, 3, 5, 64, generator=_g(9))
    dst = torch.randn(n, 3, 5, 128, generator=_g(10))
    inputs, cs = {IN: src, 2: dst}, {IN: 64, 2: 128}
    res = -1
    if form == "addend":
        inputs[3], cs[3], res = torch.randn(n, 3, 5, 96, generator=_g(11)), 96, 3
    elif form == "inplace":
        res = 2
    op = dict(kind=SLICE, src=IN, dst=2, res=res, relu=relu, p=(s0, d0, width, r0))
    m, _keep = _table(st, (3, 5), [op], [], 2, 128, cs)
    frames = _frames(n, 5, 9, 3)
    _, bufs = _run(cuda, m, frames, {b: t.to(cuda) for b, t in inputs.items()})
    _, ref = R.interpret_cnn_tables(m, st.vals, frames, dtype=torch.float32, bufs=inputs)
    assert torch.equal(R.bits(bufs[2]), R.bits(ref[2].contiguous()))
    assert torch.equal(bufs[2][..., :d0], dst[..., :d0]) and torch.equal(bufs[2][..., d0 + width:], dst[..., d0 + width:])
    _check_neighbours(cuda, m, frames, {b: t.to(cuda) for b, t in inputs.items()}, [2], float("nan"))


@pytest.mark.parametrize("hw", [(1, 1), (3, 5), (4, 4)])
@pytest.mark.parametrize("inplace", [False, True])
def test_upsample_add_bit_for_bit(cuda, hw, inplace):
    st = Store(cuda, F16)
    n = 2
    h, w = hw
    small = torch.randn(n, h, w, 64, generator=_g(12))
    big = torch.randn(n, 2 * h, 2 * w, 64, generator=_g(13))
    dst = 2 if inplace else 3
    mid = [dict(kind=CROP, src=0, dst=5, p=(0, 0, h, w)), dict(kind=SHAPE, src=5, dst=IN, p=(64,)),
           dict(kind=UPADD, src=IN, dst=dst, res=2)]
    m, _keep = _table(st, (2 * h, 2 * w), mid, [], dst, 64, {2: 64})
    frames = _frames(n, 4 * h - 1, 4 * w - 1, 3)
    inputs = {IN: small.to(cuda), 2: big.to(cuda)}
    _, bufs = _run(cuda, m, frames, inputs)
    want = big + small.repeat_interleave(2, 1).repeat_interleave(2, 2)
    assert torch.equal(R.bits(bufs[dst]), R.bits(want.contiguous()))
    _check_neighbours(cuda, m, frames, inputs, [dst], float("nan"))


@pytest.mark.parametrize("C_,s0", [(4, 8), (256, 4), (256, 0)])
@pytest.mark.parametrize("relu", [0, 1])
def test_affine_vs_float64(cuda, C_, s0, relu):
    """act(src[..., s0 : s0 + C] * a + b): one fma, so within half an ulp of the float64 value."""
    st = Store(cuda, F16)
    n = 2
    a, b = torch.randn(C_, generator=_g(14)), torch.randn(C_, generator=_g(15))
    wp, bp = st.dense(a, b)
    x = torch.randn(n, 4, 6, 264, generator=_g(16)) * 3
    m, _keep = _table(st, (4, 6), [dict(kind=AFFINE, conv=1, src=IN, dst=2, relu=relu, p=(s0,))],
                      [dict(w=wp, b=bp, cin=C_, cout=C_, cout_pad=C_, k=1, stride=1, pad=0, kpad=C_)], 2, C_, {IN: 264})
    frames = _frames(n, 7, 11, 3)
    _, bufs = _run(cuda, m, frames, {IN: x.to(cuda)})
    want = x[..., s0:s0 + C_].double() * a.double() + b.double()
    want = torch.relu(want) if relu else want
    assert bufs[2].shape == (n, 4, 6, C_) and not torch.isnan(bufs[2]).any()
    assert bool(((bufs[2].double() - want).abs() <= U * want.abs()).all())
    _check_neighbours(cuda, m, frames, {IN: x.to(cuda)}, [2], float("nan"))


@pytest.mark.parametrize("mc", [1, 32, 33, 68])
@pytest.mark.parametrize("width,s0,d0", [(4, 8, 16), (33, 3, 5), (256, 0, 16)])
def test_maskmul_vs_float64(cuda, mc, width, s0, d0):
    """dst[..., d0 : d0 + w] = src[..., s0 : s0 + w] * sum_{c < mc} mask[..., c]: each lane sums ceil(mc / 32) values,
    five shuffles add the lanes, one product: (ceil(mc / 32) + 6) u relative to |src| sum |mask|."""
    st = Store(cuda, F16)
    n = 2
    src = torch.randn(n, 5, 3, 264, generator=_g(17))
    dst = torch.randn(n, 5, 3, 272, generator=_g(18))
    mask = torch.rand(n, 5, 3, 72, generator=_g(19))
    mask[..., mc:] = float("nan")                    # channels past mc are never read
    inputs = {IN: src, 2: dst, 3: mask}
    m, _keep = _table(st, (5, 3), [dict(kind=MASKMUL, src=IN, dst=2, res=3, p=(s0, d0, width, mc))], [], 2, 272,
                      {IN: 264, 2: 272, 3: 72})
    frames = _frames(n, 9, 5, 3)
    _, bufs = _run(cuda, m, frames, {b: t.to(cuda) for b, t in inputs.items()})
    msum = mask[..., :mc].double().sum(-1, keepdim=True)
    want = src[..., s0:s0 + width].double() * msum
    got = bufs[2][..., d0:d0 + width].double()
    bound = (math.ceil(mc / 32) + 6) * U * src[..., s0:s0 + width].double().abs() * msum.abs()
    e = float(((got - want).abs() / bound.clamp(min=1e-30)).max())
    print(f"maskmul mc {mc} width {width}: error / bound {e:.2f}")
    assert e <= 1.0
    assert torch.equal(bufs[2][..., :d0], dst[..., :d0]) and torch.equal(bufs[2][..., d0 + width:], dst[..., d0 + width:])
    _check_neighbours(cuda, m, frames, {b: t.to(cuda) for b, t in inputs.items()}, [2], float("nan"))


# ---------------------------------------------------------------------------------------------------------------------
# GAP
@pytest.mark.parametrize("hw", [(1, 1), (7, 7), (56, 56)])
@pytest.mark.parametrize("div", [0, 1, 4])
def test_gap_vs_float64(cuda, hw, div):
    """out[:, c0 : c0 + C] = mean / max(div, 1), then a second GAP accumulates (p1) the same columns; the map is a
    64-real / 128-stored conv output whose stored channels 64..127 hold non-zero values the pool must ignore; the
    columns outside [c0, c0 + 64) keep their NaN.  Bound: the sequential fp32 sum of hw values and the product with
    the rounded 1 / (hw div): (hw + 3) u mean |x| / div, plus u of the accumulated sum."""
    st = Store(cuda, F16)
    n, c0 = 3, 8
    cv = _conv_entry(st, 128, 64, 128, 1, 1, 0, 21, junk_rows=True)
    mid = [dict(kind=CONV, conv=1, src=IN, dst=2, relu=0), dict(kind=GAP, src=2, p=(c0, 0, div))]
    x = torch.randn(n, hw[0], hw[1], 128, generator=_g(20)) + 0.5
    m, _keep = _table(st, hw, mid, [cv], 2, c0 + 64 + 8, {IN: 128}, gap_p=(c0, 1, 2))
    frames = _frames(n, 2 * hw[0] - 1, 2 * hw[1] - 1, 3)
    out, bufs = _run(cuda, m, frames, {IN: x.to(cuda)})
    y = bufs[2].double()
    assert bool((y[..., 64:] != 0).any()), "the padded channels should hold values the pool ignores"
    mean, amean = y[..., :64].mean(dim=(1, 2)), y[..., :64].abs().mean(dim=(1, 2))
    d = max(div, 1)
    want = mean / d + mean / 2
    bound = (hw[0] * hw[1] + 3) * U * amean * (1.0 / d + 0.5) + U * want.abs()
    got = out[:, c0:c0 + 64].double()
    e = float(((got - want).abs() / bound).max())
    print(f"gap {hw} div {div}: error / bound {e:.2f}")
    assert e <= 1.0
    assert bool(torch.isnan(out[:, :c0]).all() and torch.isnan(out[:, c0 + 64:]).all())
    bad = x.clone()
    bad[0] = float("nan")
    out2, _ = _run(cuda, m, frames, {IN: bad.to(cuda)})
    assert torch.equal(R.bits(out2[1:]), R.bits(out[1:])) and bool(torch.isnan(out2[0, c0:c0 + 64]).all())


# ---------------------------------------------------------------------------------------------------------------------
# SE and CBAM: fp32 bounds from the reduction lengths (worst case, elementwise, float64):
#   a mean over hw values              (hw + 1) u mean |y|
#   a dense layer over K inputs        |W| e_in + (K + 1) u (|W| |in| + |b|)          (ReLU is 1-Lipschitz)
#   sigmoid (expf, add, divide)        e / 4 + 4 u sigmoid
#   the product / fma of the output    e_g |y| + 2 u (|g y| + |res|)
def _se_case(cuda, C_, hw, seed):
    st = Store(cuda, F16)
    n, R_ = 2, C_ // 16
    g = _g(seed)
    wd, bd = torch.randn(R_, C_, generator=g) / math.sqrt(C_), 0.1 * torch.randn(R_, generator=g)
    wu, bu = torch.randn(C_, R_, generator=g) / math.sqrt(R_), torch.randn(C_, generator=g)
    bu[::4] = 30.0                                   # gates saturating at 1 ...
    bu[1::4] = -30.0                                 # ... and at 0
    dn, up = st.dense(wd, bd), st.dense(wu, bu)
    ent = lambda wb, ci, co: dict(w=wb[0], b=wb[1], cin=ci, cout=co, cout_pad=co, k=1, stride=1, pad=0, kpad=ci)  # noqa
    y = torch.randn(n, hw[0], hw[1], C_, generator=g) + 0.3
    r = torch.randn(n, hw[0], hw[1], C_, generator=g)
    m, _keep = _table(st, hw, [dict(kind=SE, conv=1, k=2, src=IN, dst=2, res=2, relu=1)],
                      [ent(dn, C_, R_), ent(up, R_, C_)], 2, C_, {IN: C_, 2: C_})
    frames = _frames(n, 2 * hw[0] - 1, 2 * hw[1] - 1, 3)
    inputs = {IN: y.to(cuda), 2: r.to(cuda)}
    _, bufs = _run(cuda, m, frames, inputs)
    _, ref = _ref(m, st, frames, {IN: y, 2: r})
    yd, rd = y.double(), r.double()
    hwn = hw[0] * hw[1]
    z, za = yd.mean(dim=(1, 2)), yd.abs().mean(dim=(1, 2))
    ez = (hwn + 1) * U * za
    Wd, Wu = wd.double(), wu.double()
    d = torch.relu(z @ Wd.T + bd.double())
    ed = ez @ Wd.abs().T + (C_ + 1) * U * (z.abs() @ Wd.abs().T + bd.double().abs())
    gate = torch.sigmoid(d @ Wu.T + bu.double())
    ea = ed @ Wu.abs().T + (R_ + 1) * U * (d @ Wu.abs().T + bu.double().abs())
    eg = ea / 4 + 4 * U * gate
    bound = eg[:, None, None] * yd.abs() + 2 * U * ((gate[:, None, None] * yd).abs() + rd.abs())
    e = float(((bufs[2].double() - ref[2]).abs() / bound).max())
    print(f"se C {C_} hw {hw}: error / bound {e:.3f}")
    assert e <= 1.0 and not torch.isnan(bufs[2]).any()
    assert float(gate.max()) > 1 - 1e-12 and float(gate.min()) < 1e-12, "gates saturating at both ends"
    _check_neighbours(cuda, m, frames, inputs, [2], float("nan"))


@pytest.mark.parametrize("C_,hw", [(256, (56, 56)), (512, (7, 7)), (1024, (1, 1)), (2048, (7, 7))])
def test_se_vs_float64(cuda, C_, hw):
    """Squeeze-and-excitation (segment mean, se_mlp_kernel, se_apply_kernel) with the shortcut updated in place
    (res == dst, as the SENet tables run it)."""
    _se_case(cuda, C_, hw, C_ + hw[0])


@pytest.mark.parametrize("hw,C_,inplace", [((1, 1), 256, False), ((2, 3), 32, False), ((7, 7), 512, True),
                                           ((8, 8), 256, False), ((4, 16), 32, True)])
def test_cbam_vs_float64(cuda, hw, C_, inplace):
    """CBAM + shortcut + ReLU (cbam_kernel) on maps up to the 64-position limit, including maps smaller than the 7 x 7
    spatial kernel."""
    st = Store(cuda, F16)
    n, R_ = 2, max(C_ // 16, 2)
    g = _g(C_ + hw[1])
    w1, b1 = torch.randn(R_, C_, generator=g) / math.sqrt(C_), 0.1 * torch.randn(R_, generator=g)
    w2, b2 = torch.randn(C_, R_, generator=g) / math.sqrt(R_), torch.randn(C_, generator=g)
    wsp, bsp = torch.randn(98, generator=g) * 0.3, torch.randn(1, generator=g)
    l1, l2, sp = st.dense(w1, b1), st.dense(w2, b2), st.dense(wsp, bsp)
    ent = lambda wb, ci, co, k=1: dict(w=wb[0], b=wb[1], cin=ci, cout=co, cout_pad=co, k=k, stride=1, pad=0,  # noqa
                                       kpad=ci)
    y = torch.randn(n, hw[0], hw[1], C_, generator=g)
    r = torch.randn(n, hw[0], hw[1], C_, generator=g)
    dst = 2 if inplace else 3
    m, _keep = _table(st, hw, [dict(kind=CBAM, conv=1, src=IN, dst=dst, res=2, p=(2, 3))],
                      [ent(l1, C_, R_), ent(l2, R_, C_), ent(sp, 2, 1, k=7)], dst, C_, {IN: C_, 2: C_})
    frames = _frames(n, 2 * hw[0] - 1, 2 * hw[1] - 1, 3)
    inputs = {IN: y.to(cuda), 2: r.to(cuda)}
    _, bufs = _run(cuda, m, frames, inputs)
    _, ref = _ref(m, st, frames, {IN: y, 2: r})
    yd, rd, hwn = y.double(), r.double(), hw[0] * hw[1]
    W1, W2 = w1.double(), w2.double()
    avg, mx = yd.mean(dim=(1, 2)), yd.amax(dim=(1, 2))
    eavg = (hwn + 1) * U * yd.abs().mean(dim=(1, 2))
    ha, hm = torch.relu(avg @ W1.T + b1.double()), torch.relu(mx @ W1.T + b1.double())
    eha = eavg @ W1.abs().T + (C_ + 1) * U * (avg.abs() @ W1.abs().T + b1.double().abs())
    ehm = (C_ + 1) * U * (mx.abs() @ W1.abs().T + b1.double().abs())
    hs = ha + hm
    a = hs @ W2.T + 2 * b2.double()
    ea = (eha + ehm + U * hs) @ W2.abs().T + (R_ + 2) * U * (hs @ W2.abs().T + 2 * b2.double().abs())
    cg = torch.sigmoid(a)
    ecg = ea / 4 + 4 * U * cg
    y1 = yd * cg[:, None, None]
    ey1 = yd.abs() * ecg[:, None, None] + U * y1.abs()
    comp = torch.stack((y1.amax(-1), y1.mean(-1)), 1)
    ecomp = torch.stack((ey1.amax(-1), ey1.mean(-1) + (C_ + 1) * U * y1.abs().mean(-1)), 1)
    wk = wsp.double().reshape(1, 2, 7, 7)
    s = F.conv2d(comp, wk, bsp.double(), padding=3)
    es = F.conv2d(ecomp, wk.abs(), padding=3) + 99 * U * (F.conv2d(comp.abs(), wk.abs(), padding=3) + abs(float(bsp)))
    sg = torch.sigmoid(s)[:, 0, :, :, None]
    esg = (es / 4)[:, 0, :, :, None] + 4 * U * sg
    bound = ey1 * sg + y1.abs() * esg + 2 * U * ((y1 * sg).abs() + rd.abs())
    e = float(((bufs[dst].double() - ref[dst]).abs() / bound).max())
    print(f"cbam hw {hw} C {C_}: error / bound {e:.3f}")
    assert e <= 1.0 and not torch.isnan(bufs[dst]).any()
    _check_neighbours(cuda, m, frames, inputs, [dst], float("nan"))


# ---------------------------------------------------------------------------------------------------------------------
# refusals: no launch, out_feats untouched
def test_unrunnable_tables_are_refused_before_any_launch(cuda):
    """The tables mer_cnn_workspace_bytes refuses make mer_cnn_forward return the error with no kernel launched and
    out_feats untouched.  Their weights and biases are real zeroed device buffers, and the planner's verdict is asserted
    before the forward call, so a table the planner wrongly accepted fails an assertion, never a launch on bad memory."""
    lib, fwd = _lib()
    wbuf = torch.zeros(1 << 20, dtype=torch.uint8, device=cuda)     # >= 192 x 192 split-bf16 values
    bbuf = torch.zeros(4096, dtype=torch.uint8, device=cuda)        # >= 192 fp32 biases
    frames = torch.zeros(2, 3, 3, 3, dtype=torch.uint8, device=cuda)
    ws = torch.zeros(1 << 24, dtype=torch.uint8, device=cuda)
    out = torch.full((2, 256), float("nan"), device=cuda)
    for name, m, _keep, msg in R.cnn_refused_tables(wbuf.data_ptr(), bbuf.data_ptr()):
        assert lib.mer_cnn_workspace_bytes(C.byref(m), 2) == -1, name
        before = L.launch_count()
        rc = fwd(C.byref(m), L.ptr(frames), 2, L.ptr(ws), ws.numel(), L.ptr(out), L.stream_ptr())
        torch.cuda.synchronize()
        assert rc != 0 and msg in L.lib().mer_last_error().decode(), name
        assert L.launch_count() == before and bool(torch.isnan(out).all()), name


# ---------------------------------------------------------------------------------------------------------------------
# fixed graphs
def _al(v):
    return (v + 255) & ~255


def _f16_chain_resnet18(enc, x):
    """The network after the stem in float64 over the packed (fp16-exact) weights, on a float64 stem output."""
    t = [v.cpu() for v in enc.pk.tensors]
    wb = [(t[2 * i].float(), t[2 * i + 1].float()) for i in range(20)]
    cv = [enc.model.convs[i] for i in range(20)]

    def conv(v, i, res=None, relu=True):
        c = cv[i]
        y, _ = R.cnn_conv(v[..., :c.cin], wb[i][0], wb[i][1], c.k, c.stride, c.pad)
        y = y if res is None else y + res
        return torch.relu(y) if relu else y
    x = F.max_pool2d(x.permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1)
    ci = 1
    for stage in range(4):
        for blk in range(2):
            down = stage > 0 and blk == 0
            t1 = conv(x, ci)
            ident = conv(x, ci + 2, relu=False) if down else x
            x = conv(t1, ci + 1, res=ident)
            ci += 3 if down else 2
    return x


# The fp16 operands of the 19 convolutions after the stem (each rounds its input activations to 11 bits) against the
# float64 chain on the same fp16 weights: max |pre-pool - float64| / max |float64| measured 6.9e-4 (n = 1) and 9.6e-4
# (n = 5) on an H100 80GB HBM3; the bar leaves a 4x margin over the larger.
RESNET_PREPOOL_BAR = 4e-3


@pytest.mark.parametrize("n", [1, 5])
def test_resnet18_stem_and_prepool_maps_vs_float64(cuda, n):
    """mer_resnet18_forward leaves the stem output [n, 112, 112, 128] in its first buffer and the last [n, 7, 7, 512]
    map in its second: the stem at the GEMM bar against the operand-exact fp16 reference (channels 64..127 exactly
    0), the pre-pool map against a float64 chain over the packed weights."""
    from mertools_b200 import synthetic as S
    enc = En.ResNet18Encoder(S.resnet18_state_dict(seed=6), device=cuda)
    lib = L.lib()
    total = lib.mer_resnet18_workspace_bytes(n)
    a0 = _al(n * 112 * 112 * 128 * 4)
    assert total == a0 + 2 * _al(n * 56 * 56 * 128 * 4) + _al(n * 28 * 28 * 128 * 4) + \
        _al(max(n * 112 * 112 * 192 * 2, n * 56 * 56 * 576 * 2)) + _al((n + 1) * 4)
    frames = _frames(n, 224, 224, 40 + n)
    ws = torch.full((total // 4,), float("nan"), device=cuda)
    out = torch.full((n, 512), float("nan"), device=cuda)
    fr = torch.from_numpy(frames).to(cuda)
    L.check(enc._fwd(C.byref(enc.model), L.ptr(fr), n, L.ptr(ws), total, L.ptr(out), L.stream_ptr()))
    torch.cuda.synchronize()
    stem = ws[:n * 112 * 112 * 128].view(n, 112, 112, 128).cpu().double()
    pre = ws[a0 // 4:a0 // 4 + n * 49 * 512].view(n, 7, 7, 512).cpu().double()
    x = R.stem_operand(frames, 0.00392156862745098, list(enc.IMAGENET_MEAN), list(enc.IMAGENET_STD))
    t = [v.cpu() for v in enc.pk.tensors[:2]]
    y, a = R.cnn_conv(x, t[0].float(), t[1].float(), 7, 2, 3, R.GEMM_F16)
    e = float(((stem - torch.relu(y)).abs() / a.clamp(min=1e-30)).max())
    assert e < BAR and bool((stem[..., 64:] == 0).all())
    ref = _f16_chain_resnet18(enc, torch.relu(y))
    e2 = float((pre - ref).abs().max() / ref.abs().max())
    print(f"resnet18 n {n}: stem normalised error {e:.2e}, pre-pool max error / max {e2:.2e}")
    assert not torch.isnan(pre).any() and e2 < RESNET_PREPOOL_BAR
    assert torch.allclose(out.cpu().double(), pre.mean(dim=(1, 2)), rtol=0, atol=1e-5 * float(pre.abs().max()))


@pytest.mark.parametrize("edges", [False, True])
def test_vggish_pool4_and_fc1_vs_float64(cuda, edges):
    """mer_vggish_forward leaves the pool4 map [n, 6, 4, 512] in its second buffer and fc1_1's output in its fifth.
    pool4 against a float64 stack on split operands; fc1_1 at the GEMM bar from the GPU's own pool4.  edges: examples
    non-zero only in their first and last rows and columns, what a slip of the one-channel gather would corrupt."""
    from mertools_b200 import synthetic as S
    n = 3
    enc = En.VggishEncoder(S.vggish_state_dict(seed=8), device=cuda)
    total = L.lib().mer_vggish_workspace_bytes(n)
    offs = [0]
    for sz in (n * 96 * 64 * 128 * 4, n * 48 * 32 * 128 * 4, n * 48 * 32 * 576 * 4, n * 12288 * 4, n * 4096 * 4):
        offs.append(offs[-1] + _al(sz))
    assert total == offs[-1]
    x = torch.randn(n, 96, 64, generator=_g(30)) * 2 - 1
    if edges:
        keep = torch.zeros(96, 64, dtype=torch.bool)
        keep[0], keep[-1], keep[:, 0], keep[:, -1] = True, True, True, True
        x = x * keep
    ws = torch.full((total // 4,), float("nan"), device=cuda)
    out = torch.full((n, 128), float("nan"), device=cuda)
    xd = x.to(cuda)
    L.check(enc._fwd(C.byref(enc.model), L.ptr(xd), n, L.ptr(ws), total, L.ptr(out), L.stream_ptr()))
    torch.cuda.synchronize()
    pool4 = ws[offs[1] // 4:offs[1] // 4 + n * 6 * 4 * 512].view(n, 6, 4, 512).cpu()
    fc1 = ws[offs[4] // 4:offs[4] // 4 + n * 4096].view(n, 4096).cpu()
    t = enc.pk.tensors
    wb = []
    for i in range(9):
        hi, lo = R.split_halves(t[2 * i].cpu())
        wb.append((hi.double() + lo.double(), t[2 * i + 1].cpu().double()))
    h = x[..., None]
    for i in range(6):
        c = enc.model.convs[i]
        h, _ = R.cnn_conv(h.float() if i == 0 else h, wb[i][0], wb[i][1], 3, 1, 1,
                          R.GEMM_BF16X3 if i == 0 else None)
        h = torch.relu(h)
        if i in (0, 1, 3, 5):
            h = F.max_pool2d(h.permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
        h = h[..., :c.cout] if i < 5 else h
    e = float((pool4.double() - h).abs().max() / h.abs().max())
    # fc1_1 from the GPU's own pool4, split operands without lo lo
    ph, pl = R.split_bf16(pool4.reshape(n, -1))
    wh, wl = R.split_bf16(wb[6][0].float())
    y = ph.double() @ (wh.double() + wl.double()).T + pl.double() @ wh.double().T + wb[6][1]
    a = ph.double().abs() @ (wh.double().abs() + wl.double().abs()).T + pl.double().abs() @ wh.double().abs().T + \
        wb[6][1].abs()
    e2 = float(((fc1.double() - torch.relu(y)).abs() / a).max())
    print(f"vggish edges={edges}: pool4 max error / max {e:.2e}, fc1_1 normalised error {e2:.2e}")
    assert e < 1e-4 and e2 < BAR and not torch.isnan(fc1).any()
