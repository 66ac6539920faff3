"""Reference weights for the GPU tests, written by __graft_entry__.build() into oracle/_ref/ (kept out of git): the
StyleGAN-V I3D's shipped state_dict (evaluation/common_metrics_on_video_quality/fvd/styleganv/i3d_torchscript.pt) as a
plain state_dict file.  Without the reference tree nothing is written and the tests that need the file skip."""
import os

import torch

from oracle.ref_loader import REF_ROOT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STYLEGANV_OUT = os.path.join(ROOT, "oracle", "_ref", "i3d_styleganv.pt")
STYLEGANV_SRC = os.path.join(REF_ROOT, "evaluation", "common_metrics_on_video_quality", "fvd", "styleganv",
                             "i3d_torchscript.pt")


def write_styleganv_weights() -> bool:
    if not os.path.isfile(STYLEGANV_SRC):
        return False
    sd = {k: v.clone() for k, v in torch.jit.load(STYLEGANV_SRC, map_location="cpu").state_dict().items()}
    os.makedirs(os.path.dirname(STYLEGANV_OUT), exist_ok=True)
    torch.save(sd, STYLEGANV_OUT)
    return True
