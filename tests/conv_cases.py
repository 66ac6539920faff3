"""Cases, a host model of the 3xTF32 scheme and float64 references for omt_conv3d (csrc/i3d.cu).

test_conv_cases_cpu.py checks the case list, the operand families and the error bound on the CPU;
test_gpu_conv_precision.py runs the kernel on them.

* Cases come from the networks' own tables: fvd.ARCH / BRANCHES (SAME padding, and the StyleGAN-V I3D's F.pad tables of
  its strided conv), fid.STEM / BLOCKS and quality.SLICES, de-duplicated by (Cs, Cout, kernel, stride, front padding).
  Spatial sizes are shrunk (the size does not change the kernel's path) except in the tile-walk cases, whose row counts
  give each persistent CTA 1 to 4 tiles.  Concat-branch convs keep their column offset and row width.
* The host model restates the kernel's arithmetic: A is split per element into tf32 hi = tf32_rn(a) (layout.tf32_round,
  bit-identical to tc_ptx.cuh's tf32_rn) and lo = a - hi; W arrives split the same way at pack time.  Each k-step forms
  A_lo.W_hi + A_hi.W_lo + A_hi.W_hi; lo.lo is never formed.  The tensor core reads an fp32 lo operand as tf32, i.e.
  without its low 13 mantissa bits (tf32_read).  Variants drop one correction product.
* Split-grid operands make every product and partial sum exact in fp32 with non-zero lo parts, so the kernel's result is
  unique and fp64 computes it bit for bit.  Realistic operands (post-ReLU inputs, He-scaled weights, a folded-BatchNorm
  sized bias) are compared with fp64 under an error normalised by the l2 norm of each output's products.
"""
from typing import List, NamedTuple, Optional, Tuple

import torch
import torch.nn.functional as F

from omnitokenizer_b200 import fid, fvd, quality
from omnitokenizer_b200 import layout as L

PROMOTE = 2                 # i3d.cu: k-blocks per tensor-core accumulator chunk
KB = 32                     # K per k-block
H100_SMS = 132              # SMs of an H100 SXM; the GPU test passes the device's own count
LO_STEP = 2.0 ** -12        # split-grid lo quantum: below tf32's half ulp at 1, so tf32_rn(hi + lo) = hi
MAX_PRODUCTS = 240          # non-zero weight taps per output channel of a split-grid case
# |y - y64| / sqrt(sum (x w)^2 + b^2) of the 3xTF32 result on realistic operands.  The scheme's own error (lo.lo and
# the tf32 reads of the lo operands, 2^-21 of a product at most) and the fp32 accumulation stay near 1e-6 of that norm;
# a dropped correction product leaves about 2^-12 of every product, 1e-4 and more.  test_conv_cases_cpu.py shows both
# sides of the bound on every case.
L2_BOUND = 1e-5


class ConvCase(NamedTuple):
    name: str
    B: int
    cin: int
    Cs: int                         # input channel stride (4 for the RGB input, else a multiple of 32)
    cout: int
    k: Tuple[int, int, int]
    s: Tuple[int, int, int]
    front: Tuple[int, int, int]     # front padding per axis
    dims: Tuple[int, int, int]      # input T, H, W
    out: Tuple[int, int, int]       # output To, Ho, Wo
    col: int                        # first output column in the row
    ldy: int                        # output row width (floats)

    @property
    def taps(self) -> int:
        return self.k[0] * self.k[1] * self.k[2]

    @property
    def K(self) -> int:
        return L.round_up(self.taps * 4, KB) if self.Cs == 4 else self.taps * self.Cs

    @property
    def num_kb(self) -> int:
        return self.K // KB

    @property
    def bn(self) -> int:
        return 64 if self.cout <= 64 else 128

    @property
    def M(self) -> int:
        return self.B * self.out[0] * self.out[1] * self.out[2]

    @property
    def tiles(self) -> int:
        return -(-self.M // 128) * -(-self.cout // self.bn)

    @property
    def key(self):
        return (self.Cs, self.cout, self.k, self.s, self.front)

    @property
    def id(self) -> str:
        k, s, f = ("x".join(map(str, v)) for v in (self.k, self.s, self.front))
        return f"{self.name}-{self.Cs}to{self.cout}_k{k}s{s}p{f}_M{self.M}_col{self.col}"

    def back(self) -> Tuple[int, ...]:
        """Back padding per axis that makes the output exactly `out` (negative: the last inputs are not read)."""
        return tuple((o - 1) * s + k - n - f for o, s, k, n, f in zip(self.out, self.s, self.k, self.dims, self.front))


def _out(n, k, s, front, back):
    return (n + front + back - k) // s + 1


def _i3d_case(name, cin, cout, k, s, dims, col, ldy, front=None, B=1):
    kk, ss = (k,) * 3, (s,) * 3
    if front is None:
        front, out = fvd.same_geometry(kk, ss, dims)
    else:
        front, back = front
        out = tuple(_out(n, k, s, f, b) for n, f, b in zip(dims, front, back))
    return ConvCase(name, B, cin, fvd.cpad(cin), cout, kk, ss, tuple(front), tuple(dims), tuple(out), col,
                    ldy or cout)


def i3d_cases() -> List[ConvCase]:
    """Every Unit3D of fvd.ARCH: the stem at odd sizes (SAME pads 3 in front) and at the StyleGAN-V I3D's F.pad tables
    (both temporal parities), every Inception branch unit with its concat column."""
    out = []
    for name, kind, spec in fvd.ARCH:
        if kind == "unit":
            cin, cout, k, s = spec
            out.append(_i3d_case(name, cin, cout, k, s, (9, 21, 19) if s > 1 else (3, 9, 7), 0, None))
            if name in fvd.STYLEGANV_PADS:
                for t, tab in zip((10, 9), fvd.STYLEGANV_PADS[name][2]):
                    fr, bk = (tab[4], tab[2], tab[0]), (tab[5], tab[3], tab[1])
                    out.append(_i3d_case(name + "-sgv", cin, cout, k, s, (t, 20, 18), 0, None, front=(fr, bk)))
        elif kind == "mixed":
            cin, w = spec
            total = w[0] + w[2] + w[4] + w[5]
            offs = {"b0": 0, "b1b": w[0], "b2b": w[0] + w[2], "b3b": w[0] + w[2] + w[4]}
            for b, (wi, k, src) in fvd.BRANCHES.items():
                c_in = cin if src in ("x", "p") else w[fvd.BRANCHES[src][0]]
                if b in offs:
                    out.append(_i3d_case(f"{name}.{b}", c_in, w[wi], k, 1, (3, 9, 7), offs[b], fvd.cpad(total)))
                else:
                    out.append(_i3d_case(f"{name}.{b}", c_in, w[wi], k, 1, (3, 9, 7), 0, None))
    return out


def _conv2d_case(name, cin, cout, kh, kw, s, ph, pw, hw, col, ldy, B=1):
    out = tuple(fid.out_size(n, k, s, p) for n, k, p in zip(hw, (kh, kw), (ph, pw)))
    return ConvCase(name, B, cin, fvd.cpad(cin), cout, (1, kh, kw), (1, s, s), (0, ph, pw), (1,) + tuple(hw),
                    (1,) + out, col, ldy or fvd.cpad(cout))


def fid_cases() -> List[ConvCase]:
    """Every BasicConv2d of fid.STEM / BLOCKS (kernel depth 1), concat branches at their column of the block's row."""
    out = []
    for c in fid.STEM:
        if isinstance(c, fid.Conv):
            out.append(_conv2d_case(c.name, c.cin, c.cout, *c.k, c.s, *c.p, (17, 15), 0, None))
    for name, convs, _, cout in fid.BLOCKS:
        for c in convs:
            col, ldy = (0, None) if c.col is None else (c.col, fvd.cpad(cout))
            out.append(_conv2d_case(f"{name}.{c.name}", c.cin, c.cout, *c.k, c.s, *c.p, (17, 15), col, ldy))
    return out


def vgg_cases() -> List[ConvCase]:
    """The 13 3x3 convs of quality.SLICES (pad 1, rows of exactly cout floats), two images per launch."""
    return [_conv2d_case(f"vgg{c.idx}", c.cin, c.cout, 3, 3, 1, 1, 1, (12, 10), 0, c.cout, B=2)
            for convs in quality.SLICES for c in convs]


def walk_cases(sms: int = H100_SMS) -> List[ConvCase]:
    """Tile counts S - 1, S + 1, 2S + 1 and 3S + 1 (S = SMs; one CTA per SM): each CTA walks 1 to 4 tiles, on both
    tile widths, with a partial last row tile.  A 3x3 conv on 32 channels: 9 k-blocks, one chunk short of PROMOTE."""
    out = []
    for tiles, cout in ((sms - 1, 64), (sms + 1, 128), (2 * sms + 1, 128), (3 * sms + 1, 48)):
        rows = tiles * 128 - 37
        h = 16
        w = -(-rows // h)
        while (h * w + 127) // 128 != tiles:
            w -= 1
        out.append(_conv2d_case(f"walk{tiles}", 32, cout, 3, 3, 1, 1, 1, (h, w), 0, None))
    return out


def network_cases() -> List[ConvCase]:
    """i3d_cases + fid_cases + vgg_cases, de-duplicated by key; of equal keys the first that writes a column slice
    (or else the first) is kept."""
    seen = {}
    for c in i3d_cases() + fid_cases() + vgg_cases():
        have = seen.get(c.key)
        if have is None or (have.col == 0 and have.ldy == have.cout and c.col > 0):
            seen[c.key] = c
    return list(seen.values())


def all_cases(sms: int = H100_SMS) -> List[ConvCase]:
    return network_cases() + walk_cases(sms)


def reduced(c: ConvCase, cout: int = 32) -> ConvCase:
    """The case at a size the host model runs quickly: at most `cout` output channels, one image, few rows."""
    dims = tuple(min(n, m) for n, m in zip(c.dims, (9 if c.k[0] > 1 and c.s[0] > 1 else 3, 13, 11)))
    out = tuple(max(1, _out(n, k, s, f, f)) for n, k, s, f in zip(dims, c.k, c.s, c.front))
    n = min(c.cout, cout)
    return c._replace(B=1, dims=dims, out=out, cout=n, col=0, ldy=n)


# ---------------------------------------------------------------- operands

def split_tf32(t: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """The kernel's split of an fp32 tensor: hi = tf32_rn(t) (round to nearest, ties away), lo = t - hi (exact)."""
    hi = L.tf32_round(t.float())
    return hi, t.float() - hi


def tf32_read(t: torch.Tensor) -> torch.Tensor:
    """An fp32 operand as the tensor core reads it in a tf32 MMA: the low 13 mantissa bits dropped."""
    return (t.float().contiguous().view(torch.int32) & -8192).view(torch.float32)


def pack(w: torch.Tensor, c: ConvCase) -> Tuple[torch.Tensor, torch.Tensor]:
    """(w_hi, w_lo) [n_pad, K] exactly as the networks pack a weight (cout, cin, kt, kh, kw): fvd.pack_weight, then
    layout.tf32_round for hi and the exact remainder for lo."""
    wp, K = fvd.pack_weight(w)
    assert K == c.K, (K, c.K)
    return split_tf32(wp)


def to_cl(x: torch.Tensor, Cs: int) -> torch.Tensor:
    """(B, C, T, H, W) -> channels-last (B, T, H, W, Cs), pad channels zero."""
    y = torch.zeros(x.shape[0], *x.shape[2:], Cs, dtype=x.dtype, device=x.device)
    y[..., :x.shape[1]] = x.permute(0, 2, 3, 4, 1)
    return y


def split_grid_operands(c: ConvCase, seed: int):
    """x (B, cin, T, H, W), w (cout, cin, kt, kh, kw), bias (cout,), fp32, with x, w = hi + lo: hi in {-1, 0, 1},
    lo in {-1, 0, 1} * 2^-12 and non-zero only where hi is, so tf32_rn(x) = hi.  Each output channel keeps at most
    MAX_PRODUCTS non-zero weight taps, so no output sums more than 3 * MAX_PRODUCTS non-zero products: every partial
    sum is a multiple of 2^-12 below 2^8, 20 significant bits.  The bias is an integer in [-4, 4]."""
    g = torch.Generator().manual_seed(seed)

    def grid(shape):
        hi = torch.randint(-1, 2, shape, generator=g).float()
        lo = torch.randint(-1, 2, shape, generator=g).float() * LO_STEP * (hi != 0)
        return hi + lo

    x = grid((c.B, c.cin) + c.dims)
    w = grid((c.cout, c.cin) + c.k).view(c.cout, -1)
    n = w.shape[1]
    if n > MAX_PRODUCTS:
        keep = torch.rand(c.cout, n, generator=g).argsort(dim=1)[:, :MAX_PRODUCTS]
        w = w * torch.zeros_like(w).scatter_(1, keep, 1.0)
    b = torch.randint(-4, 5, (c.cout,), generator=g).float()
    return x, w.view((c.cout, c.cin) + c.k), b


def realistic_operands(c: ConvCase, seed: int):
    """x: post-ReLU relu(N(0, 1)) (the RGB input: signed uniform in [-1, 1]); w: He-scaled N(0, 2 / fan_in); bias:
    N(0, 0.5^2), the size of a folded BatchNorm's beta - mean s."""
    g = torch.Generator().manual_seed(seed)
    if c.Cs == 4:
        x = torch.rand((c.B, c.cin) + c.dims, generator=g) * 2 - 1
    else:
        x = torch.randn((c.B, c.cin) + c.dims, generator=g).clamp_min(0)
    w = torch.randn((c.cout, c.cin) + c.k, generator=g) * (2.0 / (c.cin * c.taps)) ** 0.5
    b = torch.randn(c.cout, generator=g) * 0.5
    return x, w, b


# ---------------------------------------------------------------- references and the host model

def conv64(x: torch.Tensor, w: torch.Tensor, c: ConvCase, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """float64 conv3d of x (B, C, T, H, W) with w (cout, C, kt, kh, kw) at the case's padding and output size,
    channels-last (B, To, Ho, Wo, cout).  Runs on x's device."""
    fr, bk = c.front, c.back()
    xp = F.pad(x.double(), (fr[2], bk[2], fr[1], bk[1], fr[0], bk[0]))
    y = F.conv3d(xp, w.double(), None if bias is None else bias.double(), stride=c.s)
    assert tuple(y.shape[2:]) == c.out, (tuple(y.shape[2:]), c.out)
    return y.permute(0, 2, 3, 4, 1)


def split_grid_reference(x, w, b, c: ConvCase, relu: bool) -> torch.Tensor:
    """fp64 A_hi.W_hi + A_lo.W_hi + A_hi.W_lo + bias (then ReLU), cast to fp32: the one value a correct kernel gives."""
    xh, xl = split_tf32(x)
    wh, wl = split_tf32(w)
    y = conv64(xh, wh, c) + conv64(xl, wh, c) + conv64(xh, wl, c) + b.double().to(x.device)
    return (y.clamp_min(0) if relu else y).float()


PRODUCTS = ("lo_hi", "hi_lo", "hi_hi")          # A_lo.W_hi, A_hi.W_lo, A_hi.W_hi


def emulate(x, w, b, c: ConvCase, drop: Optional[str] = None) -> torch.Tensor:
    """The scheme on the host: the retained products of the split operands (lo read as tf32), summed exactly in
    float64, plus bias, rounded once to fp32 (no accumulation error).  drop: one of PRODUCTS to leave out."""
    xh, xl = split_tf32(x)
    wh, wl = split_tf32(w)
    terms = {"lo_hi": (tf32_read(xl), wh), "hi_lo": (xh, tf32_read(wl)), "hi_hi": (xh, wh)}
    y = b.double().to(x.device) + sum(conv64(a, ww, c) for p, (a, ww) in terms.items() if p != drop)
    return y.float()


def l2_scale(x, w, b, c: ConvCase) -> torch.Tensor:
    """sqrt(sum over an output's products (x w)^2 + b^2), float64, channels-last."""
    return (conv64(x.double() ** 2, w.double() ** 2, c) + b.double().to(x.device) ** 2).sqrt()


def l2_error(y: torch.Tensor, ref64: torch.Tensor, scale: torch.Tensor) -> float:
    """max |y - ref64| / scale over the outputs (y fp32, ref64 and scale float64, same shape)."""
    return float(((y.double() - ref64).abs() / scale.clamp_min(1e-30)).max())
