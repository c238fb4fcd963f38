"""VQBASE.encode_code without a GPU: the host logic above the emulated C-ABI of tests/test_host_logic_vq_cpu.py (plus the
scene-map entries of tests/test_scene_maps_cpu.py). Bit identity with the eval-mode model's own quantiser, no side effects on a
train-mode model (counters, reservoir, k-means, BatchNorm statistics, autograd), input validation, and the seg-config case
of the real reference's fixture (tests/golden/encode_code.pt). The kernels run on the GPU in tests/test_gpu_encode_code.py."""
import os

import pytest
import torch

from conftest import GOLDEN
from encode_code_common import case_input, case_model, load_fixture, sampled_err
from test_gpu_parity import _explain_index_mismatches
from test_host_logic_vq_cpu import vq_emu  # noqa: F401  (fixture)
from test_scene_maps_cpu import scene_emu  # noqa: F401  (fixture)


@pytest.fixture
def on_kernel_device(monkeypatch):
    """CPU tensors stand in for device tensors above the emulated C-ABI."""
    from models import vqvae
    monkeypatch.setattr(vqvae, "_kernel_device", lambda t: True)


def _tiny():
    from models import VQBASE
    g = torch.load(os.path.join(GOLDEN, "vqbase_tiny.pt"), weights_only=False)
    m = VQBASE(g["ddconfig"], g["n_embed"], g["embed_dim"], 10, 100)
    m.load_state_dict(g["state_dict"])
    with torch.no_grad():                    # non-default running statistics, so that using them is visible
        m.quant_conv[1].running_mean.normal_(0, 0.5, generator=torch.Generator().manual_seed(1))
        m.quant_conv[1].running_var.uniform_(0.5, 2.0, generator=torch.Generator().manual_seed(2))
    return m, g["x"]


def _eval_indices(m, x):
    """The indices the eval-mode model's own quantiser returns in a forward (grad enabled)."""
    seen = {}
    hook = m.quantize.register_forward_hook(lambda _m, _i, o: seen.__setitem__("idx", o[2].detach().clone()))
    was = m.training
    m.eval()
    m(x)
    m.train(was)
    hook.remove()
    return seen["idx"].view(-1)


def _snapshot(m):
    return ({k: v.clone() for k, v in m.state_dict().items()}, {n: mod.training for n, mod in m.named_modules()},
            m.quantize.q_counter, m.quantize.reservoir, m.quantize.reservoir.clone())


def _assert_unchanged(m, snap):
    sd, modes, q, res, res_val = snap
    now = m.state_dict()
    assert now.keys() == sd.keys()
    for k, v in sd.items():
        assert now[k].dtype == v.dtype and torch.equal(now[k], v), k
    assert {n: mod.training for n, mod in m.named_modules()} == modes
    assert m.quantize.q_counter == q
    assert m.quantize.reservoir is res and torch.equal(m.quantize.reservoir, res_val)


def test_tiny_bit_identical_to_the_eval_forward(vq_emu, on_kernel_device):
    m, x = _tiny()
    want = _eval_indices(m, x)
    first = len(vq_emu.names)
    tok = m.encode_code(x)
    assert tok.dtype == torch.int64 and tok.shape == (2, 8, 8)
    assert torch.equal(tok.flatten(), want)
    n = vq_emu.names[first:]
    # eval BatchNorm and one arg-min; no batch statistics, no k-means
    assert n.count("mas_vq_forward") == 1 and "mas_bn_invstd" in n and "mas_bn_stats" not in n and "mas_kmeans_update" not in n
    dec = m.decode_code(tok)                                    # decode_code is the inverse: a [B, 3, H, W] image again
    assert dec.shape == x.shape


@pytest.mark.parametrize("q_counter", ["warm-up", "re-init"])
def test_tiny_train_mode_has_no_side_effects(vq_emu, on_kernel_device, q_counter):
    """A train-mode model at the codebook's warm-up (Codebook.forward would return no indices) and one step before a k-means
    re-initialisation (Codebook.forward would replace the codebook), with a reservoir and deferred collection set."""
    m, x = _tiny()
    want = _eval_indices(m, x)
    m.train()
    cb = m.quantize
    cb.q_counter = 0 if q_counter == "warm-up" else cb.q_init - 1
    cb.reservoir = torch.randn(50, cb.codebook_dim, generator=torch.Generator().manual_seed(3))
    cb.defer_collect = True
    snap = _snapshot(m)
    with torch.enable_grad():
        tok = m.encode_code(x)
    assert torch.equal(tok.flatten(), want)
    assert not tok.requires_grad and tok.grad_fn is None
    _assert_unchanged(m, snap)
    assert not hasattr(cb, "_deferred_z") and cb.defer_collect is True
    assert all(p.grad is None for p in m.parameters())


def test_validation(on_kernel_device, monkeypatch):
    m, x = _tiny()
    for bad in (x.double(), x.half(), x.to(torch.int32), (x * 255).to(torch.uint8),        # dtypes (uint8: not a scene model)
                torch.zeros(2, 4, 16, 16), torch.zeros(2, 159, 16, 16),                      # channel counts
                torch.zeros(2, 3, 15, 16), torch.zeros(2, 3, 16, 18)[..., :17],              # H / W off the factor 2
                torch.zeros(0, 3, 16, 16), torch.zeros(3, 16, 16)):                          # empty, not 4-D
        with pytest.raises(ValueError):
            m.encode_code(bad)
    from models import vqvae
    monkeypatch.setattr(vqvae, "_kernel_device", lambda t: t.is_cuda)
    with pytest.raises(ValueError):                                                          # a CPU tensor
        m.encode_code(x)


def test_seg_fixture_from_compact_and_dense_maps(scene_emu, on_kernel_device):
    """The seg-config case of the reference fixture from the compact planes and from their dense map: the same tokens from both
    (the compact map is expanded into the operand the dense one is padded into), the eval latent within the fp16 operand
    rounding the emulation reproduces, and every index that differs from the reference's a Voronoi-boundary crossing of our
    own latent. No dense copy is made of the compact map."""
    from encode_code_common import recipe
    fx = load_fixture()
    c = fx["seg"]
    m = case_model(fx, "seg").eval()
    lab = case_input(fx, "seg")
    lat = {}
    hook = m.quant_conv.register_forward_hook(lambda _m, _i, o: lat.__setitem__("z", o.detach().clone()))
    with torch.no_grad():
        m.quant_conv(m.encoder(lab))                     # the eval latent, recorded by the hook
    hook.remove()
    first = len(scene_emu.names)
    tok = m.encode_code(lab)
    n = scene_emu.names[first:]
    assert torch.equal(m.encode_code(recipe.dense_map(lab)), tok)
    assert n.count("mas_scene_expand") == 1 and "mas_nchw_to_nhwc_pad" not in n
    e = sampled_err(lat["z"], c["latent"])
    assert e < 3e-3, e                                    # the GPU test's bound; measured 2.3e-3 on the first image
    E = m.quantize.embedding.weight.detach()
    zf = lat["z"].permute(0, 2, 3, 1).reshape(-1, E.shape[1])
    mism = _explain_index_mismatches(zf, E, tok.flatten(), c["idx"].flatten())
    print("seg fixture: latent error %.2e, %d of %d indices differ" % (e, mism, tok.numel()))
    assert mism <= 26, mism                               # 5 % of the 512 rows, each one checked above
