"""The per-sample float64 sums of ops.sample_sumsq and ops.sample_noise (fq_sample_sums.cuh) against a numpy restatement of
the kernels' summation order, compared bit for bit.

The inputs make every product exact in float64: y is fp32 (optionally plus a bias as one fp32 add) and q = round(y / 0.25)
* 0.25, so y^2, q^2, y * q and e^2 (e = y - q, at most 24 significant bits) all fit in 53 bits.  Each __fma_rn is then one
float64 add, and numpy adding the same terms in the same order gives the kernels' bits; the float64 sums still round, so
any other order shows."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CHUNK = 16384   # elements per (row, chunk) unit
THREADS = 256


def terms(y, q, sums):
    """the per-element float64 terms of each sum, in output column order: [sums][rows, row_len]"""
    if sums == 1:
        return [y * y]
    if sums == 2:
        return [y, y * y]
    e = y - q
    return [y, y * y, q, q * q, y * q, e, e * e]


def restate(y, q, sums, vec):
    """The kernels' order on float64 [rows, row_len] rows: [rows, sums].  A row is cut into units of CHUNK elements (one
    unit when shorter); thread t of a unit adds its vectors t, t + 256, ... of `vec` elements, in index order and
    component by component, from 0; the 32 lanes of a warp combine by s + shfl_xor(s, o) for o = 16, 8, 4, 2, 1; lane 0 of
    warps 0..7 is added in warp order; a row's units are added in unit order from unit 0."""
    rows, n = y.shape
    chunk = min(n, CHUNK)
    chunks = -(-n // chunk)
    steps = -(-chunk // (THREADS * vec))   # vectors per thread in a full unit
    lane = np.arange(32)
    out = []
    for t in terms(y, q, sums):
        a = np.zeros((rows, chunks * chunk))   # zero terms past the row's end and in unused slots add nothing
        a[:, :n] = t
        a = a.reshape(rows, chunks, chunk)
        b = np.zeros((rows, chunks, steps * THREADS * vec))
        b[:, :, :chunk] = a
        b = b.reshape(rows, chunks, steps, THREADS, vec).transpose(0, 1, 3, 2, 4).reshape(rows, chunks, THREADS, -1)
        s = np.zeros((rows, chunks, THREADS))
        for k in range(b.shape[-1]):
            s = s + b[..., k]
        s = s.reshape(rows, chunks, THREADS // 32, 32)
        for o in (16, 8, 4, 2, 1):
            s = s + s[..., lane ^ o]
        u = s[..., 0, 0]
        for w in range(1, THREADS // 32):
            u = u + s[..., w, 0]
        r = u[:, 0]
        for c in range(1, chunks):
            r = r + u[:, c]
        out.append(r)
    return np.stack(out, 1)


def memory_rows(t):
    """[rows, row_len] float64 numpy in t's memory order (channels-last read as N, H, W, C)"""
    if t.dim() == 4 and not t.is_contiguous():
        t = t.permute(0, 2, 3, 1)
    return t.reshape(t.shape[0], -1).double().cpu().numpy()


def biased(y, bias, bias_period):
    """y + bias as the one fp32 add the kernels make, in y's memory order"""
    yr = torch.from_numpy(memory_rows(y)).float()
    if bias is None:
        return yr.double().numpy()
    i = torch.arange(yr.shape[1])
    b = bias.cpu()[i // bias_period if bias_period > 0 else i % -bias_period]
    return (yr + b).double().numpy()


def vec_of(*ts):
    return 4 if ts[0][0].numel() % 4 == 0 and all(t.data_ptr() % 16 == 0 for t in ts) else 1


def quantized(y):
    return torch.round(y / 0.25) * 0.25


def misaligned(shape, g):
    n = int(np.prod(shape))
    t = torch.randn(n + 1, device="cuda", generator=g)[1:].view(shape)   # 4 bytes off 16-byte alignment
    assert t.data_ptr() % 16 != 0
    return t


SHAPES = {
    "one_chunk": lambda g: torch.randn(6, 1000, device="cuda", generator=g),
    "ragged_last_chunk": lambda g: torch.randn(4, 40000, device="cuda", generator=g),
    "twelve_element_last_chunk": lambda g: torch.randn(3, 3 * CHUNK + 12, device="cuda", generator=g),
    "scalar_row_len": lambda g: torch.randn(4, 2 * CHUNK + 3, device="cuda", generator=g),
    "scalar_misaligned": lambda g: misaligned((4, 40000), g),
    "channels_last": lambda g: torch.randn(3, 12, 56, 56, device="cuda", generator=g).contiguous(
        memory_format=torch.channels_last),
}


@pytest.mark.parametrize("name", sorted(SHAPES))
def test_sample_sumsq_order(name):
    from cnn_quantization_b200 import ops
    y = SHAPES[name](torch.Generator(device="cuda").manual_seed(11))
    want = restate(memory_rows(y), None, 1, vec_of(y))[:, 0]
    assert torch.equal(ops.sample_sumsq(y).cpu(), torch.from_numpy(want))


@pytest.mark.parametrize("with_q", [False, True])
@pytest.mark.parametrize("name", sorted(SHAPES))
def test_sample_noise_order(name, with_q):
    from cnn_quantization_b200 import ops
    y = SHAPES[name](torch.Generator(device="cuda").manual_seed(12))
    q = torch.empty_like(y).copy_(quantized(y)) if with_q else None   # y's strides: read in y's memory order
    qs = (q,) if with_q else ()
    want = torch.from_numpy(restate(memory_rows(y), memory_rows(q) if with_q else None, 7 if with_q else 2,
                                    vec_of(y, *qs)))
    for max_ctas in (0, 1, 7):
        assert torch.equal(ops.sample_noise(y, q, max_ctas=max_ctas).cpu(), want), max_ctas


@pytest.mark.parametrize("layout", ["nchw", "channels_last", "nchw_7x7", "channels_last_7x7", "scalar", "misaligned"])
def test_sample_noise_bias_order(layout):
    from cnn_quantization_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(13)
    c, hw = (12, 56) if layout in ("nchw", "channels_last") else (20, 7) if layout.endswith("7x7") else (3, 7)
    shape = (3, c, hw, hw)
    y = misaligned(shape, g) if layout == "misaligned" else torch.randn(shape, device="cuda", generator=g)
    if layout.startswith("channels_last"):
        y = y.contiguous(memory_format=torch.channels_last)
    period = -c if layout.startswith("channels_last") else hw * hw
    bias = torch.randn(c, device="cuda", generator=g) * 3
    yb = biased(y, bias, period)
    qr = np.round(yb / 0.25) * 0.25
    q = torch.empty_like(y)
    if y.data_ptr() % 16:
        q = misaligned(shape, g)
    if layout.startswith("channels_last"):
        q.permute(0, 2, 3, 1).copy_(torch.from_numpy(qr).float().view(3, hw, hw, c))
    else:
        q.copy_(torch.from_numpy(qr).float().view(shape))
    want = torch.from_numpy(restate(yb, qr, 7, vec_of(y, q)))
    for max_ctas in (0, 1, 7):
        assert torch.equal(ops.sample_noise(y, q, bias, period, max_ctas=max_ctas).cpu(), want), (layout, max_ctas)
    want2 = torch.from_numpy(restate(yb, None, 2, vec_of(y)))
    assert torch.equal(ops.sample_noise(y, None, bias, period).cpu(), want2), layout
