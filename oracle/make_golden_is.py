"""Generate tests/golden/is_inception.pt from the UNMODIFIED reference Inception Score code
(evaluation/common_metrics_on_video_quality/calculate_is.py), loaded by file path, with the installed torchvision.

Weights: oracle.is_oracle.make_state_dict (fid_oracle's seeded units, a 1000-class fc and seeded AuxLogits), with
BatchNorm statistics calibrated through torchvision's pool wiring and fc scaled (is_oracle.calibrate) on seeded frames,
so that every scored case (is_oracle.CASES) scores at least 2 (1.5 for splits of two frames, which score at most 2)
and its frames' top-1 classes differ.  calculate_is.py builds its network with
inception_v3(pretrained=True, transform_input=False): that module attribute is replaced by a function that checks
those arguments and returns torchvision's Inception3(transform_input=False, aux_logits=True, init_weights=False) with
the seeded state dict loaded strictly, so nothing is downloaded.  Hooks on that network record each batch's input
(sampled), its logits and, for the first case, each block's output (summaries); the probabilities stored are
F.softmax of those logits over the classes, the rows the reference writes into `preds`.
Cases: is_oracle.CASES.

    python -m oracle.make_golden_is
"""
import importlib.util
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F
import torchvision

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import is_oracle as io  # noqa: E402
from oracle import fid_oracle as fo  # noqa: E402
from oracle.ref_loader import REF_ROOT  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "is_inception.pt")
IS_SRC = os.path.join(REF_ROOT, "evaluation", "common_metrics_on_video_quality", "calculate_is.py")
W_SEED = 17
CAL_SEEDS = (201, 202)
LOGIT_SPREAD = 8.0


def load_module(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


class Recorder:
    """The stub for calculate_is.py's inception_v3 and what the network it returns saw."""

    def __init__(self, sd):
        self.sd, self.inputs, self.logits, self.endpoints = sd, [], [], None

    def __call__(self, pretrained=None, transform_input=None, **kw):
        assert pretrained is True and transform_input is False and not kw, (pretrained, transform_input, kw)
        net = torchvision.models.Inception3(transform_input=False, aux_logits=True, init_weights=False)
        net.load_state_dict({k: v.clone() for k, v in self.sd.items()}, strict=True)
        net.register_forward_pre_hook(self.record_input)
        net.register_forward_hook(self.record_logits)
        if self.endpoints is not None:
            for name, _, _, _ in fo.BLOCKS:
                getattr(net, name).register_forward_hook(self.endpoint_hook(name))
        return net

    # the hooks return None: a forward hook that returns a value replaces the module's output
    def record_input(self, module, args):
        self.inputs.append(args[0].detach().clone())

    def record_logits(self, module, args, out):
        self.logits.append(out.detach().clone())

    def endpoint_hook(self, name):
        def hook(module, args, out):
            if name not in self.endpoints:          # the first batch's
                self.endpoints[name] = out.detach().clone()
        return hook


def main():
    torch.manual_seed(0)
    calc = load_module("calculate_is_ref", IS_SRC)
    sd = io.make_state_dict(W_SEED)
    cal = torch.cat([io.preprocess(io.frames((4, 64, 64), CAL_SEEDS[0])),
                     io.preprocess(io.frames((2, 64, 80), CAL_SEEDS[1], lo=-1.0))])
    scale = io.calibrate(sd, cal, LOGIT_SPREAD)
    out = {"w_seed": W_SEED, "cal_seeds": CAL_SEEDS, "fingerprint": fo.conv_fingerprint(sd), "bn": fo.bn_stats(sd),
           "fc_scale": scale, "fc_bias": sd["fc.bias"].clone(), "cases": {}}
    assert all(torch.equal(v, sd[k]) for k, v in io.fixture_state_dict(out).items())
    for i, (name, spec) in enumerate(io.CASES.items()):
        rec = Recorder(sd)
        if i == 0:
            rec.endpoints = {}
        calc.inception_v3 = rec
        x, _ = io.case_input(spec)
        if spec["fn"] == "calculate_is":
            mean, std = calc.calculate_is(x, "cpu", splits=spec["splits"])
        else:
            mean, std = calc.inception_score(list(x), cuda=False, batch_size=spec["batch_size"], resize=spec["resize"],
                                             splits=spec["splits"])
        logits = torch.cat(rec.logits)
        probs = F.softmax(logits, dim=1)
        ora = io.case_probabilities(sd, spec)
        same = torch.equal(ora, probs)
        o_mean, o_std = io.inception_score(probs.double().numpy(), spec["splits"])
        top1 = probs.argmax(1)
        print(f"{name}: IS {mean:.6f} +- {std:.6f} over {probs.shape[0]} frames, {len(set(top1.tolist()))} top-1 "
              f"classes, max|logit| {float(logits.abs().max()):.2f}; oracle probabilities equal: {same}, oracle IS "
              f"rel diff {abs(o_mean - mean) / mean:.1e}")
        # a split of n rows scores at most n (n distinct one-hot rows), so splits of 2 rows are held to 1.5
        floor = min(2.0, 0.75 * (probs.shape[0] // spec["splits"]))
        if spec.get("scored", True):
            assert mean >= floor, f"{name}: IS {mean} < {floor}: the fixture would not test the score"
            assert len(set(top1.tolist())) > 1, f"{name}: every frame has the same top-1 class"
        pre = torch.cat(rec.inputs)
        g = torch.Generator().manual_seed(spec["seed"])
        pi = torch.randint(0, pre.numel(), (512,), generator=g)
        entry = {"spec": dict(spec), "logits": logits, "probs": probs, "mean": float(mean), "std": float(std),
                 "pre_shape": tuple(pre.shape), "pre_idx": pi, "pre_val": pre.flatten()[pi].clone()}
        if rec.endpoints is not None:
            entry["endpoints"] = {k: fo.endpoint_summary(v, 1000 + j) for j, (k, v) in enumerate(rec.endpoints.items())}
        out["cases"][name] = entry
    torch.save(out, OUT)
    print(f"wrote {OUT} ({os.path.getsize(OUT) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
