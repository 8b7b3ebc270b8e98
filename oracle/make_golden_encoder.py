"""ORACLE fixture (test infrastructure): the reference's BasicEncoder4 (dpvo/extractor.py, needs only torch) run once on
the CPU, so that tests/test_frontend_cpu.py can hold frontend.Encoder4 to it without a checkout of the reference.

    python oracle/make_golden_encoder.py      (needs the reference tree, see oracle/refimport.py)

Stored in tests/golden/encoder_ref.pt, float32: the input image [1, 1, 3, 29, 35] (odd sizes: partial windows of both
strided layers) and the outputs of fnet (norm 'instance', 128 channels) and inet (norm 'none', 384 channels), with the
weights of `rule_weights`, which the test recreates.
"""
import importlib.util
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

OUT = os.path.join(ROOT, "tests", "golden", "encoder_ref.pt")
IMAGE = (1, 1, 3, 29, 35)


def rule_weights(module, salt):
    """deterministic parameters by name order: weights sin(0.7 i + k) sqrt(2 / fan_in), biases 0.1 cos(1.3 i + k)"""
    with torch.no_grad():
        for k, (name, p) in enumerate(sorted(module.named_parameters())):
            i = torch.arange(p.numel(), dtype=torch.float64)
            if name.endswith("weight"):
                v = torch.sin(0.7 * i + k + salt) * math.sqrt(2.0 / (p[0].numel()))
            else:
                v = 0.1 * torch.cos(1.3 * i + k + salt)
            p.copy_(v.view_as(p).float())
    return module


def rule_image():
    i = torch.arange(math.prod(IMAGE), dtype=torch.float64).view(IMAGE)
    return (0.8 * torch.sin(0.05 * i) + 0.3 * torch.cos(0.31 * i)).float()


def main():
    path = os.path.join("/root/reference", "dpvo", "extractor.py")
    spec = importlib.util.spec_from_file_location("_ref_extractor", path)
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    x = rule_image()
    out = {"image": x}
    for nm, dim, norm, salt in (("fnet", 128, "instance", 0), ("inet", 384, "none", 100)):
        enc = rule_weights(ex.BasicEncoder4(output_dim=dim, norm_fn=norm), salt).eval()
        with torch.no_grad():
            out[nm] = enc(x).contiguous()
    torch.save(out, OUT)
    print("wrote %s (%d bytes)" % (OUT, os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
