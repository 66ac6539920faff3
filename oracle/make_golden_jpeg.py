"""Records Pillow's JPEG save and reload on the seeded grid of oracle/jpeg_oracle.py, so the oracle, jpeg.quant_tables
and omt_jpeg_roundtrip_u8 are pinned to the bytes vqgan_eval.py's img.save(path) / pytorch-fid's Image.open(path)
.convert("RGB") produce for a .jpg / .JPEG path.

    python -m oracle.make_golden_jpeg     (writes tests/golden/jpeg_roundtrip.pt; needs Pillow)

Per case of jpeg_oracle.grid(): (H, W, quality, kind, seed), the SHA-256 of the seeded input (jpeg_oracle.content) and
of Pillow's output, img.save(f, "JPEG", quality=q) then Image.open(f).convert("RGB"); the output bytes themselves for
images of at most SMALL pixels.  Also the quantisation tables Pillow writes at every quality 1..100, and the Pillow and
libjpeg-turbo versions that made the file.
"""
import hashlib
import io
import os

import numpy as np
import torch

from oracle import jpeg_oracle as J

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "jpeg_roundtrip.pt")
SMALL = 64


def sha(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def pillow_roundtrip(rgb: np.ndarray, quality: int):
    """Pillow's save to JPEG and reload: (output (H, W, 3) uint8, the file's quantisation tables [2, 64])."""
    from PIL import Image
    f = io.BytesIO()
    Image.fromarray(rgb).save(f, "JPEG", quality=quality)
    f.seek(0)
    im = Image.open(f)
    tables = np.array([im.quantization[0], im.quantization[1]], dtype=np.int64)
    return np.asarray(im.convert("RGB")), tables


def versions() -> dict:
    import PIL
    from PIL import features
    return {"pillow": PIL.__version__, "libjpeg_turbo": features.version("libjpeg_turbo")}


def main():
    cases = []
    for H, W, q, kind, seed in J.grid():
        x = J.content(kind, H, W, seed)
        y, _ = pillow_roundtrip(x, q)
        case = {"H": H, "W": W, "quality": q, "kind": kind, "seed": seed, "input_sha": sha(x), "output_sha": sha(y)}
        if H * W <= SMALL:
            case["output"] = torch.from_numpy(y.copy())
        cases.append(case)
    tables = torch.from_numpy(np.stack([pillow_roundtrip(np.zeros((8, 8, 3), np.uint8), q)[1]
                                        for q in range(1, 101)]).astype(np.int32))
    torch.save({"cases": cases, "tables": tables, "versions": versions()}, OUT)
    print(f"wrote {OUT}: {len(cases)} cases, {versions()}")


if __name__ == "__main__":
    main()
