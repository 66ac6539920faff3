"""CPU numerics model of the fp16 hi/lo-split tensor-core path (OMT_MATH=f16x3) inside the oracle: every tensor-core
product a.b is replaced by  hi(a).hi(b) + 2^-11 (hi(a).lo'(b) + lo'(a).hi(b)),  hi = fp16(x), lo' = fp16((x - hi) * 2^11),
products exact, fp32 accumulation.  Prints flipped code indices and decoder pixel error per golden case, next to the
3xTF32 model the shipped kernels implement and the single-product f16x1 model (tests/f16x1_model.py: row-scaled fp16 hi
operands, one product, fp32 accumulation)."""
import sys, os
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from oracle import omni_oracle as oo
from util import load_golden, golden_setup, check_sub
from f16x1_model import mm_f16x1


def _tf32_rna(x):
    return ((x.contiguous().view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)
def _tf32_trunc(x):
    return (x.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)
def mm_3xtf32(a, b):
    ah, bh = _tf32_rna(a), _tf32_rna(b)
    al, bl = _tf32_trunc(a - ah), _tf32_trunc(b - bh)
    return (al @ bh + ah @ bl) + ah @ bh
def split16(x):
    hi = x.clamp(-65504, 65504).half()
    lo = ((x - hi.float()) * 2048.0).half()
    return hi.float(), lo.float()
def mm_f16x3(a, b):
    ah, al = split16(a); bh, bl = split16(b)
    return ah @ bh + (ah @ bl + al @ bh) * (1.0 / 2048.0)
def mm_f16x2(a, b):      # weights-only / activation-only variants for curiosity
    ah, al = split16(a); bh, bl = split16(b)
    return ah @ bh + (ah @ bl) * (1.0 / 2048.0)

names = sys.argv[1:] or ["img64", "vid5x64", "vid9x128_b2", "img256_cfg1", "cnn_vid5x64"]
for name in names:
    fx = load_golden(name)
    cfg, sd, x = golden_setup(fx)
    is_image = x.ndim == 4
    if "idx" not in fx:
        continue
    with torch.no_grad():
        for label, model in (("3xtf32", mm_3xtf32), ("f16x3", mm_f16x3), ("f16x2", mm_f16x2), ("f16x1", mm_f16x1)):
            oo.MATMUL_MODEL = model
            emb, idx = oo.encode(sd, cfg, x, include_embeddings=True)
            rec = oo.decode(sd, cfg, fx["idx"].long(), is_image)
            flips = int((idx != fx["idx"].long()).sum())
            err = check_sub(fx["rec"], rec, 1.0, "rec")
            print(f"{name:14s} {label:7s} flips {flips}/{idx.numel()}  max|dpx| {err:.2e}", flush=True)
    oo.MATMUL_MODEL = None
