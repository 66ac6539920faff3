"""CPU numerics model of the f16x1 math mode, and the near-tie test that tells a flipped code the mode may cause from a
real error.

Model (oracle.omni_oracle.MATMUL_MODEL): every tensor-core product a @ b becomes ONE fp16 product.  Each row of a is
multiplied by the power of two that puts its largest magnitude in [2^14, 2^15), b by one such power of two per matrix;
both are rounded to fp16 (round to nearest even) and the products, exact in fp32, are summed in fp32.  The scales come
off exactly afterwards.
"""
import torch


def _pow2_scale(mx: torch.Tensor) -> torch.Tensor:
    """2^(14 - floor(log2 mx)): maps mx into [2^14, 2^15); 1 where mx == 0."""
    _, e = torch.frexp(mx)                       # mx = m 2^e, m in [0.5, 1): floor(log2 mx) = e - 1
    return torch.where(mx > 0, torch.exp2((15 - e).to(mx.dtype)), torch.ones_like(mx))


def mm_f16x1(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """a @ b as the f16x1 kernels form it (module docstring); b may be batched, one scale per matrix."""
    a, b = a.float(), b.float()
    sa = _pow2_scale(a.abs().amax(dim=-1, keepdim=True))
    sb = _pow2_scale(b.abs().amax(dim=(-2, -1), keepdim=True))
    ah = (a * sa).clamp(-65504, 65504).half().float()
    bh = (b * sb).clamp(-65504, 65504).half().float()
    return (ah @ bh) / sa / sb


def provable_near_tie(z_ref, z_new, E, a, b, slack: float = 1e-5) -> torch.Tensor:
    """For rows whose code moved from a (the reference's, at z_ref) to b (at z_new): True where the move is explained by
    the change of z alone.  With d(z, E) = |z|^2 - 2 z.E + |E|^2, moving z to z' changes the gap d(z, E_b) - d(z, E_a)
    by 2 (z - z').(E_a - E_b), at most 2 |z' - z| |E_a - E_b| in magnitude.  So b can win at z' only if the gap at z_ref
    is within that bound; `slack` covers the fp32 rounding of the distances on either side."""
    z, zn, E = z_ref.double(), z_new.double(), E.double()
    Ea, Eb = E[a], E[b]
    gap = ((z - Eb) ** 2).sum(-1) - ((z - Ea) ** 2).sum(-1)
    bound = 2.0 * (zn - z).norm(dim=-1) * (Ea - Eb).norm(dim=-1)
    return gap <= bound + slack
