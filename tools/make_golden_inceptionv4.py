#!/usr/bin/env python
"""Regenerate tests/golden/inceptionv4_reference.npz from a checkout of the reference repository.

    DEAR_REFERENCE_DIR=<reference checkout> python tools/make_golden_inceptionv4.py

The fixture holds what the reference's own Inception-v4 class (dear/inceptionv4.py) computes: the shapes of its
state_dict in order, and its logits on a seeded input after loading the seeded weights that
tests/test_models.py::test_inceptionv4_matches_the_reference_file builds with our model (same seed, same BatchNorm
perturbation, same order of random draws).  Rerun it if torch's initialisation draws ever change.
"""
import importlib.util
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from dear_pytorch_b200.models.registry import create  # noqa: E402


def main():
    ref_dir = os.environ.get("DEAR_REFERENCE_DIR", "")
    path = os.path.join(ref_dir, "dear", "inceptionv4.py")
    if not (ref_dir and os.path.isfile(path)):
        sys.exit("DEAR_REFERENCE_DIR must name a checkout of the reference (dear/inceptionv4.py not found)")
    spec = importlib.util.spec_from_file_location("_ref_inceptionv4", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    # the test's draws, in the test's order: our model's init, the BatchNorm perturbation, then the input
    torch.manual_seed(0)
    ours = create("inceptionv4").eval()
    with torch.no_grad():
        for m in ours.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.running_mean.normal_(0, 0.1); m.running_var.uniform_(0.5, 1.5); m.weight.uniform_(0.5, 1.5); m.bias.normal_(0, 0.1)
    x = torch.randn(1, 3, 299, 299)
    ref = mod.InceptionV4(num_classes=1000).eval()
    src, mine = ref.state_dict(), ours.state_dict()
    shapes = [list(v.shape) for v in src.values()]
    if shapes != [list(v.shape) for v in mine.values()]:
        sys.exit("the state_dicts do not line up tensor for tensor")
    ref.load_state_dict(dict(zip(src.keys(), mine.values())))
    with torch.no_grad():
        logits = ref(x)
    out = os.path.join(ROOT, "tests", "golden", "inceptionv4_reference.npz")
    np.savez_compressed(out, logits=logits.numpy().astype(np.float32), shapes=np.array([json.dumps(shapes)]))
    print("wrote", out)


if __name__ == "__main__":
    main()
