"""LPIPS drop-in (losses/lpips.py) without a GPU: parameter layout and seeded parameters against the real reference
(tests/golden/lpips.pt), resolution of `losses.lpips` next to a reference checkout, and the refusals of what has no
kernel. The kernels and the module's numbers are tested on the GPU (tests/test_gpu_lpips.py)."""
import hashlib
import os
import subprocess
import sys
import textwrap

import pytest
import torch

from conftest import GOLDEN, PKG
from lpips_common import build_lpips, golden_tool, seeded_lpips


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(GOLDEN, "lpips.pt"), weights_only=False)


def _sha(t):
    return hashlib.sha256(t.detach().contiguous().numpy().tobytes()).hexdigest()


@pytest.mark.parametrize("name", ["256", "72"])
def test_state_dict_and_seeded_parameters_match_reference(golden, name):
    case = golden[name]
    m, checks = seeded_lpips(case)
    sd = m.state_dict()
    assert list(sd) == list(case["init"])
    assert list(sd)[:3] == ["scaling_layer.shift", "scaling_layer.scale", "vgg.slice1.0.weight"]
    assert list(sd)[-1] == "lin4.model.1.weight" and "vgg.slice5.5.bias" in sd
    for k, v in sd.items():
        ref = case["init"][k]
        assert tuple(v.shape) == ref["shape"] and str(v.dtype) == ref["dtype"], k
        assert _sha(v) == ref["sha256"], k
    assert checks == case["fill_checks"]
    assert all(not p.requires_grad for p in m.parameters())
    real, fake = golden_tool.images(case["seed"], case["size"], case["batch"])
    assert _sha(torch.cat([real, fake])) == case["images_sha256"]


def test_checkpoint_loads_in_both_directions(golden):
    m, _ = seeded_lpips(golden["72"])
    m2 = build_lpips()
    m2.load_state_dict(m.state_dict())
    for (k, a), (_, b) in zip(m.state_dict().items(), m2.state_dict().items()):
        assert torch.equal(a, b), k


def test_refuses_training_mode_and_trainable_parameters():
    m = build_lpips()
    x = torch.zeros(1, 3, 16, 16)
    m.train()
    with pytest.raises(RuntimeError, match=r"\.eval\(\)"):
        m(x, x)
    m.eval()
    m.lin2.model[1].weight.requires_grad_(True)
    with pytest.raises(RuntimeError, match="no weight gradients"):
        m(x, x)


def test_lpips_resolves_to_ours_and_lpips_with_object_subclasses_it(tmp_path):
    ref = tmp_path / "ref" / "losses"
    ref.mkdir(parents=True)
    (ref / "__init__.py").write_text("")
    (ref / "lpips.py").write_text("raise ImportError('the reference lpips must not be picked up')\n")
    (ref / "lpips_with_object.py").write_text(textwrap.dedent("""
        from .lpips import LPIPS


        class LPIPSWithObject(LPIPS):
            def forward(self, real_x, fake_x, object_boxes):
                return super().forward(real_x, fake_x)
    """))
    prog = textwrap.dedent("""
        import sys
        sys.path[:0] = [%r, %r]
        import losses.lpips as lp
        assert lp.__file__.startswith(%r)
        assert "torchvision" not in sys.modules
        import losses.lpips_with_object as lo
        assert lo.__file__.startswith(%r)
        assert issubclass(lo.LPIPSWithObject, lp.LPIPS) and lo.LPIPS is lp.LPIPS
        print("ok")
    """) % (PKG, str(tmp_path / "ref"), PKG, str(tmp_path / "ref"))
    r = subprocess.run([sys.executable, "-c", prog], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stderr
