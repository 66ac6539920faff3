"""Writes tests/golden/jpeg_decode.pt: small seeded JPEG files as Pillow writes them (jpeg_decode_oracle.matrix over
the sizes up to 31 x 33) and the sha256 of Pillow's Image.open(f).convert("RGB") bytes of each, with the Pillow and
libjpeg-turbo versions that made them.

    python -m oracle.make_golden_jpeg_decode
"""
import hashlib
import os

import torch
from PIL import __version__ as pil_version, features

from oracle import jpeg_decode_oracle as D

SMALL = [s for s in D.SIZES if s[0] * s[1] <= 31 * 33]


def main():
    files, shas, cases = [], [], []
    for H, W, sub, q, kind, seed, opts in D.matrix(SMALL):
        data = D.fixture(H, W, sub, q, kind, seed, **opts)
        files.append(data)
        shas.append(hashlib.sha256(D.pillow_rgb(data).tobytes()).hexdigest())
        cases.append((H, W, sub, q, kind, seed, sorted(opts)))
    path = os.path.join(os.path.dirname(__file__), "..", "tests", "golden", "jpeg_decode.pt")
    torch.save({"files": files, "sha256": shas, "cases": cases, "pillow": pil_version,
                "libjpeg_turbo": features.version("libjpeg_turbo")}, path)
    print(f"{len(files)} files, {sum(map(len, files))} bytes -> {path}")


if __name__ == "__main__":
    main()
