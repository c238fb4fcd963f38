"""Shared by the VQBASE.encode_code tests: the fixture (tests/golden/encode_code.pt, written from the real reference by
tools/make_golden_encode_code.py), the recipe's own input and codebook generators (loaded by path), and the drop-in VQBASE of
a fixture case built the way the recipe built the reference's: seeded constructor, the recorded running statistics, the
codebook rebuilt bit for bit from the recorded base latents and noise seed."""
import importlib.util
import os

import torch

from conftest import GOLDEN, ROOT

_spec = importlib.util.spec_from_file_location("make_golden_encode_code", os.path.join(ROOT, "tools", "make_golden_encode_code.py"))
recipe = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(recipe)


def load_fixture():
    return torch.load(os.path.join(GOLDEN, "encode_code.pt"), weights_only=False)


def case_model(fx, name):
    """The drop-in VQBASE of fixture case `name` on the CPU, in train mode (as constructed)."""
    from models import VQBASE
    c = fx[name]
    torch.manual_seed(c["weight_seed"])
    m = VQBASE(c["ddconfig"], c["n_embed"], c["embed_dim"], c["init_steps"], c["reservoir_size"])
    checks = {k: (float(p.detach().double().sum()), float(p.detach().double().abs().sum())) for k, p in m.named_parameters()}
    assert checks == c["param_checks"]                  # the reference's seeded init, parameter for parameter
    with torch.no_grad():
        m.quant_conv[1].running_mean.copy_(c["running_mean"])
        m.quant_conv[1].running_var.copy_(c["running_var"])
        m.quantize.embedding.weight.copy_(recipe.codebook(c["base"], c["n_embed"], c["noise_seed"]))
    assert recipe.sha(m.quantize.embedding.weight) == c["codebook_sha256"]
    return m


def case_input(fx, name):
    """The recorded batch on the CPU: fp32 images (img) or the compact scene planes (seg; recipe.dense_map expands them)."""
    x = recipe.inputs(name, fx[name]["x_seed"])
    assert recipe.sha(x) == fx[name]["input_sha256"]
    return x


def sampled_err(t, rec, images=None):
    """Norm-wise relative error of t's strided sample against a recorded one (recipe.sample); images=k: only the samples
    that fall in the first k images of the batch."""
    got = t.detach().reshape(-1).cpu()
    if images is not None:
        got = got[:images * got.numel() // rec["shape"][0]]
    got = got[::rec["stride"]].double()
    want = rec["val"][:got.numel()].double()
    return float((got - want).norm() / want.norm())
