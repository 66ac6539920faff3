"""The persistent f16 spatial attention core (csrc/attention_f16.cu) across its work-item walk.

The kernel puts one CTA on each SM and walks the work items (128-query tile, head, sequence) with a static stride; a
producer warp streams each item's K / V tiles through a 4-stage ring and fetches the next item's Q while the consumer
warpgroups finish the current one.  These tests sweep the item count T over 1, S - 1, S, S + 1, 2S + 1 and 3S + 1 (S the
SM count) so that the CTAs run 1 to 4 items, at N = 128 (2 key tiles, fewer than the ring has stages) and at N = 4096
(64 key tiles, the long-sequence shape).  Every output sits in a sentinel-filled buffer with guard rows and a leading
dimension wider than the heads; the guard bits must survive.  Three launches must agree bit for bit, one launch must
equal launches on windows of its sequences bit for bit, and the result must match fp64 softmax attention.
"""
import pytest
import torch

from omnitokenizer_b200 import layout as L

pytestmark = pytest.mark.gpu

SENT32 = 0x7FBADBAD          # fp32 NaN pattern of the fp32 output buffer
SENT16 = 0x7E5B              # fp16 NaN pattern of the O plane buffers
PRE, POST = 3, 5             # guard rows before and after every output
T_KEYS = {"1": lambda s: 1, "S-1": lambda s: s - 1, "S": lambda s: s, "S+1": lambda s: s + 1,
          "2S+1": lambda s: 2 * s + 1, "3S+1": lambda s: 3 * s + 1}


def _cabi():
    from omnitokenizer_b200 import _cabi
    _cabi.load()
    return _cabi


def _sms():
    return _cabi().device_info()[0]


def _static_planes(x, ps):
    xs = x.float() * ps
    hi = xs.clamp(-65504, 65504).half()
    return hi.view(torch.int16), (xs - hi.float()).half().view(torch.int16)


class Problem:
    """q, k unit-norm x per-dim scale as the QKV epilogue leaves them, v rows of very different magnitude (the operand
    construction of test_gpu_f16x3.py::test_attn_spatial_h).  ramp: key norms grow along each sequence, so the row
    maxima keep rising from key tile to key tile."""

    def __init__(self, nseq, N, H, seed, dev, ramp=False):
        self.nseq, self.N, self.H, self.M = nseq, N, H, nseq * N
        M = self.M
        g = torch.Generator().manual_seed(seed)
        q = torch.nn.functional.normalize(torch.randn(M, H, 64, generator=g), dim=-1) * (torch.rand(64, generator=g) + 0.5)
        k = torch.nn.functional.normalize(torch.randn(M, H, 64, generator=g), dim=-1) * (torch.rand(64, generator=g) + 0.5)
        if ramp:
            k = k * (0.1 + 2.4 * (torch.arange(M) % N).float() / N)[:, None, None]
        v = torch.randn(M, H, 64, generator=g) * torch.logspace(-2, 2, M)[torch.randperm(M, generator=g)][:, None, None]
        self.q, self.k, self.v = q, k, v
        self.qs, self.ks = L.pow2_scale(float(q.abs().max())), L.pow2_scale(float(k.abs().max()))
        qh, ql = _static_planes(q.reshape(M, H * 64), self.qs)
        kh, kl = _static_planes(k.reshape(M, H * 64), self.ks)
        vh, vl, vinv = L.split_rows_rs(v.reshape(M * H, 64))
        vh, vl, vinv = vh.reshape(M, H * 64), vl.reshape(M, H * 64), vinv.reshape(M, H).t()
        self.planes = [t.contiguous().to(dev) for t in (qh, ql, kh, kl, vh, vl)]
        self.vinv = vinv.contiguous().to(dev)           # [H][M]

    def run(self, o=None, o_hi=None, o_lo=None, ldo=None, s0=0, s1=None):
        """Launch on sequences [s0, s1): the planes at row s0 N, vinv as its own [H][rows] block."""
        s1 = self.nseq if s1 is None else s1
        r0, r1 = s0 * self.N, s1 * self.N
        ld = self.H * 64
        qh, ql, kh, kl, vh, vl = (t[r0:r1] for t in self.planes)
        vinv = self.vinv[:, r0:r1].contiguous()
        _cabi().call("omt_attn_spatial_h", qh, ql, ld, kh, kl, ld, vh, vl, ld, vinv, self.qs * self.ks, o, o_hi, o_lo,
                     ldo, s1 - s0, self.N, self.H, 8.0)

    def reference(self, dev):
        """fp64 softmax(8 q k^T) v, [M, H * 64]."""
        shp = (self.nseq, self.N, self.H, 64)
        qq, kk, vv = (t.view(shp).permute(0, 2, 1, 3).to(dev, torch.float64) for t in (self.q, self.k, self.v))
        out = torch.empty(self.nseq, self.H, self.N, 64, dtype=torch.float64, device=dev)
        for s in range(self.nseq):
            out[s] = torch.softmax((qq[s] @ kk[s].transpose(-1, -2)) * 8.0, dim=-1) @ vv[s]
        return out.permute(0, 2, 1, 3).reshape(self.M, self.H * 64)


def _f32_buf(rows, ld, dev):
    b = torch.empty(PRE + rows + POST, ld, device=dev)
    b.view(torch.int32).fill_(SENT32)
    return b


def _f16_buf(rows, ld, dev):
    return torch.full((2, PRE + rows + POST, ld), SENT16, dtype=torch.int16, device=dev)


def _check_guards(buf, rows, cols, sent):
    bits = buf.view(torch.int32) if buf.dtype == torch.float32 else buf
    assert bool((bits[..., :PRE, :] == sent).all()), "guard rows before the output were written"
    assert bool((bits[..., PRE + rows:, :] == sent).all()), "guard rows after the output were written"
    assert bool((bits[..., PRE:PRE + rows, cols:] == sent).all()), "columns beyond the heads were written"


def _check_accuracy(o, want, N, what):
    """test_attn_spatial_h's bound of 2e-5 (N <= 1024); the fp32 sums over the keys (P''.V and the row sum) gather
    rounding error at most in proportion to their length, so 4096 keys get 3x that bound."""
    assert not bool(torch.isnan(o).any()), f"{what}: NaN left inside the output"
    rel = ((o.double() - want).abs() / want.abs().amax(dim=1, keepdim=True).clamp_min(1e-3)).max().item()
    assert rel < (2e-5 if N <= 1024 else 6e-5), f"{what}: max error relative to the row magnitude {rel:.2e}"


def _walk(p, dev, what):
    """Launch into guarded fp32 and plane buffers three times; check guards, determinism, accuracy and the planes."""
    cols = p.H * 64
    ldo = cols + 8
    runs = []
    for _ in range(3):
        buf = _f32_buf(p.M, ldo, dev)
        p.run(o=buf[PRE:], ldo=ldo)
        torch.cuda.synchronize()
        _check_guards(buf, p.M, cols, SENT32)
        runs.append(buf)
    for b in runs[1:]:
        assert torch.equal(b.view(torch.int32), runs[0].view(torch.int32)), f"{what}: launches differ"
    o = runs[0][PRE:PRE + p.M, :cols]
    _check_accuracy(o, p.reference(dev), p.N, what)
    op = _f16_buf(p.M, ldo, dev)
    p.run(o_hi=op[0, PRE:], o_lo=op[1, PRE:], ldo=ldo)
    torch.cuda.synchronize()
    _check_guards(op, p.M, cols, SENT16)
    got = L.join_f16(op[0, PRE:PRE + p.M, :cols].cpu(), op[1, PRE:PRE + p.M, :cols].cpu())
    assert (got - o.cpu()).abs().max().item() <= 2.0 ** -21 * o.abs().max().item(), f"{what}: O planes"


@pytest.mark.parametrize("T", list(T_KEYS))
def test_item_counts_n128(cuda, T):
    """N = 128: one query tile and two key tiles per (sequence, head); T = n_seq x heads work items."""
    items = T_KEYS[T](_sms())
    H = next(h for h in (8, 4, 2, 1) if items % h == 0)
    p = Problem(items // H, 128, H, 300 + items, cuda)
    _walk(p, cuda, f"N=128 items={items} heads={H}")


@pytest.mark.parametrize("ramp", [False, True])
def test_long_sequences_n4096(cuda, ramp):
    """N = 4096 (the long-sequence shape): 32 query tiles and 64 key tiles per (sequence, head), 8 heads, 2 sequences
    -> 512 work items, about 4 per CTA."""
    p = Problem(2, 4096, 8, 77, cuda, ramp=ramp)
    _walk(p, cuda, f"N=4096 ramp={ramp}")


def test_placement_invariance(cuda):
    """One launch with at least 2S + 1 items equals launches on windows of its sequences, bit for bit: every item decodes
    to the same (query tile, head, sequence) whichever CTA runs it, and no item reads another sequence's K / V."""
    N, H = 256, 8
    per_seq = H * N // 128
    nseq = (2 * _sms() + 1 + per_seq - 1) // per_seq + 1
    p = Problem(nseq, N, H, 91, cuda, ramp=True)
    cols = p.H * 64
    whole = torch.empty(p.M, cols, device=cuda)
    p.run(o=whole, ldo=cols)
    windows = [(0, 1), (1, 4), (4, nseq - 1), (nseq - 1, nseq)]
    parts = torch.empty(p.M, cols, device=cuda)
    for s0, s1 in windows:
        p.run(o=parts[s0 * N:], ldo=cols, s0=s0, s1=s1)
    torch.cuda.synchronize()
    assert torch.equal(whole.view(torch.int32), parts.view(torch.int32))
