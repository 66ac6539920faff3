"""The host checks of the bilinear clip entry points other than omt_resample_clips (tests/test_gpu_clip_ingest.py checks
that one): omt_fvd_preprocess, omt_fid_preprocess, omt_fvd_suite_preprocess, omt_is_preprocess and omt_eval_downsample
in each input form.  From one valid call, one descriptor field, table entry or argument at a time is made bad; each
such call must raise a RuntimeError naming its entry point before any launch, so the output keeps its sentinel.  The
entry points without a flip or a window must also refuse both.  The valid call then gives the same bytes as before."""
import re

import pytest
import torch

from omnitokenizer_b200 import _cabi
from omnitokenizer_b200 import metricnet as M

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
B, F, H, W, OH, OW = 2, 3, 20, 24, 12, 14
# omt_clip_desc words: 0-1 src, 2 H, 3 W, 4 y0, 5 x0, 6 wh, 7 ww, 8 rh, 9 rw, 10 cy, 11 cx, 12 flip, 13 tv, 14 th, 15 form
CASES = {   # name -> (entry point, form, source layout, has a byte table, takes a flip and a window)
    "fvd": ("omt_fvd_preprocess", None, "u8", True, True),
    "fid": ("omt_fid_preprocess", None, "u8", True, True),
    "suite_u8": ("omt_fvd_suite_preprocess", M.FORM_U8, "u8", False, False),
    "suite_f32": ("omt_fvd_suite_preprocess", M.FORM_F32, "fchw", False, False),
    "suite_f32_trunc": ("omt_fvd_suite_preprocess", M.FORM_F32_TRUNC, "fchw", False, False),
    "is_u8": ("omt_is_preprocess", M.FORM_U8, "u8", False, False),
    "is_f32": ("omt_is_preprocess", M.FORM_F32, "fchw", False, False),
    "eval_u8": ("omt_eval_downsample", 1, "u8", True, False),          # OMT_DS_U8
    "eval_f32": ("omt_eval_downsample", 0, "cfhw", False, False),      # OMT_DS_F32
}


class Call:
    """One valid call of a case on B clips of F frames of H x W, resized to OH x OW.  The source holds one clip more
    than the call reads, so a descriptor may grow its frame by a row or a column and stay inside it."""

    def __init__(self, case):
        self.name, self.form, layout, table, self.windows = CASES[case]
        frames = 1 if self.name == "omt_fid_preprocess" else F
        g = torch.Generator().manual_seed(0)
        if layout == "u8":
            shape = (B + 1, frames, H, W, 3)
            self.src = torch.randint(0, 256, shape, generator=g, dtype=torch.uint8).to(DEV)
        else:
            shape = (B + 1, frames, 3, H, W) if layout == "fchw" else (B + 1, 3, frames, H, W)
            self.src = (torch.rand(shape, generator=g) * 1.2 - 0.6).to(DEV)
        self.src_elems = self.src.numel()
        self.clip_elems = self.src_elems // (B + 1)
        self.desc_host = M.clip_descs(B, self.clip_elems, H, W, OH, OW)
        self.tab_host = M.axis_tables(H, W, OH, OW)
        self.desc, self.tab = self.desc_host.to(DEV), self.tab_host.to(DEV)
        self.lut = (M.byte_lut()[0] * (255 if self.name == "omt_fvd_preprocess" else 1)).to(DEV) if table else None
        if self.name == "omt_eval_downsample":
            self.out = torch.empty(B, frames, OH, OW, 3, dtype=torch.uint8, device=DEV)
        else:
            self.out = torch.empty(B, frames, OH, OW, 4, device=DEV)
        self.sentinel = 7 if self.out.dtype == torch.uint8 else -7.0

    def __call__(self, src=..., src_elems=None, desc=None, tab=None, lut=...):
        src = self.src if src is ... else src
        lut = self.lut if lut is ... else lut
        src_elems = self.src_elems if src_elems is None else src_elems
        desc = self.desc if desc is None else desc
        tab = self.tab if tab is None else tab
        tables = (desc, self.desc_host, tab, self.tab_host, self.tab_host.numel())
        if self.name == "omt_fvd_preprocess":
            args = (src, src_elems, *tables, lut, None, B, F, OH, OW)
        elif self.name == "omt_fid_preprocess":
            args = (src, src_elems, *tables, lut, None, B, OH, OW)
        elif self.name == "omt_fvd_suite_preprocess":
            args = (src, src_elems, self.form, 3, *tables, B, F, OH, OW)
        elif self.name == "omt_is_preprocess":
            args = (src, src_elems, self.form, *tables, B, F, OH, OW)
        else:
            args = (src, src_elems, self.form, *tables, lut, None, B, F, OH, OW)
        _cabi.call(self.name, *args, self.out)

    def refused(self, msg, **kw):
        """The call with kw raises a RuntimeError naming the entry point and msg, and leaves the output alone."""
        self.out.fill_(self.sentinel)
        with pytest.raises(RuntimeError, match=f"{self.name}: .*{re.escape(msg)}"):
            self(**kw)
        torch.cuda.synchronize()
        assert bool((self.out == self.sentinel).all()), f"{self.name}: a refused call wrote its output"


@pytest.mark.parametrize("case", list(CASES))
def test_checks_refuse_bad_input_before_launch(case, cuda):
    c = Call(case)
    c()
    torch.cuda.synchronize()
    want = c.out.clone()
    d, t = c.desc_host[1], c.tab_host
    for row, word, value, msg in ((d, 2, 1 << 20, "outside the"), (d, 4, 1, "window"), (d, 10, OH, "crop"),
                                  (d, 12, 2, "flip / form"), (d, 15, 2, "flip / form"),
                                  (d, 13, 1 << 20, "vertical table"), (d, 14, 2, "horizontal table"),
                                  (t, 1, 1000, "indices outside")):
        saved = int(row[word])
        row[word] = value
        c.refused(msg)
        row[word] = saved
    c.refused("outside the", src_elems=B * c.clip_elems - 1)
    c.refused("null", src=None)
    if c.lut is not None:
        c.refused("null" if c.name != "omt_eval_downsample" else "byte table", lut=None)
    c.refused("aligned", desc=c.desc.data_ptr() + 4)
    c.refused("aligned", tab=c.tab.data_ptr() + 4)
    if not c.windows:
        # a flip, and a window origin inside a frame one row or one column larger: only the missing flip and window
        # refuse them
        for changes in ({12: 1}, {2: H + 1, 4: 1}, {3: W + 1, 5: 1}):
            for word, value in changes.items():
                d[word] = value
            c.refused("no flip and no window")
            d[2:] = M.clip_descs(B, c.clip_elems, H, W, OH, OW)[1, 2:]
    assert torch.equal(c.desc_host, M.clip_descs(B, c.clip_elems, H, W, OH, OW))
    c.out.fill_(c.sentinel)
    c()
    torch.cuda.synchronize()
    assert torch.equal(c.out.view(torch.uint8), want.view(torch.uint8))
