"""VQBASE.encode_code on the H100: tokens bit-identical to the eval-mode model's own quantiser on every route, agreement with
the real reference (tests/golden/encode_code.pt, tools/make_golden_encode_code.py), no side effects on a train-mode model,
input validation, the chain into MakeAScene (seg / image tokens -> generate / score -> decode_code), and the round trip
decode_code(encode_code(x)) against the eval forward."""
import os

import pytest
import torch
import torch.nn.functional as F

from conftest import GOLDEN, rel_err
from encode_code_common import case_input, case_model, load_fixture, recipe, sampled_err
from test_gpu_parity import _explain_index_mismatches

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
TINY = dict(z_channels=32, in_channels=3, out_channels=3, channels=[32, 32, 64], num_res_blocks=1, resolution=16,
            attn_resolutions=[8], dropout=0.0)


@pytest.fixture(scope="module")
def fx():
    return load_fixture()


@pytest.fixture(scope="module")
def img_model(fx):
    return case_model(fx, "img").to(DEV)


@pytest.fixture(scope="module")
def seg_model(fx):
    return case_model(fx, "seg").to(DEV)


def _eval_quantiser(m, x):
    """(latent after BatchNorm, indices) of the eval-mode model's own forward, from hooks; the module's mode is restored."""
    seen = {}
    hz = m.quant_conv.register_forward_hook(lambda _m, _i, o: seen.__setitem__("z", o.detach()))
    hi = m.quantize.register_forward_hook(lambda _m, _i, o: seen.__setitem__("idx", o[2].detach()))
    was = m.training
    m.eval()
    try:
        m.encode(x)
    finally:
        m.train(was)
        hz.remove(); hi.remove()
    return seen["z"], seen["idx"].view(-1)


def _images(b, size=256, seed=0):
    return (torch.rand(b, 3, size, size, generator=torch.Generator().manual_seed(seed)) * 2 - 1).to(DEV)


# ------------------------------------------------------------------------------------------------ bit identity
@pytest.mark.parametrize("b", [1, 2, 7, 32])
def test_img_config_bit_identical_to_the_eval_quantiser(img_model, b):
    x = _images(b, seed=b)
    tok = img_model.encode_code(x)
    assert tok.dtype == torch.int64 and tok.shape == (b, 16, 16) and tok.device == x.device
    assert torch.equal(tok.flatten(), _eval_quantiser(img_model, x)[1])


def test_tiny_config_simt_route_bit_identical():
    from mas_b200 import _lib, ops
    from models import VQBASE
    g = torch.load(os.path.join(GOLDEN, "vqbase_tiny.pt"), weights_only=False)
    m = VQBASE(g["ddconfig"], g["n_embed"], g["embed_dim"], 10, 100)
    m.load_state_dict(g["state_dict"])
    m.to(DEV)
    x = g["x"].to(DEV)
    ops.set_impl(_lib.IMPL_SIMT)
    try:
        l0 = _lib.launch_count()
        tok = m.encode_code(x)
        torch.cuda.synchronize()
        assert _lib.launch_count() > l0
        assert torch.equal(tok.flatten(), _eval_quantiser(m, x)[1])
    finally:
        ops.set_impl(_lib.IMPL_AUTO)


def test_seg_config_compact_and_dense_bit_identical(fx, seg_model):
    lab = case_input(fx, "seg").to(DEV)
    dense = recipe.dense_map(lab.cpu()).to(DEV)
    tok_c, tok_d = seg_model.encode_code(lab), seg_model.encode_code(dense)
    assert tok_c.shape == (2, 16, 16)
    assert torch.equal(tok_c, tok_d)
    assert torch.equal(tok_c.flatten(), _eval_quantiser(seg_model, lab)[1])
    assert torch.equal(tok_d.flatten(), _eval_quantiser(seg_model, dense)[1])


# ------------------------------------------------------------------------------------------------ against the reference
@pytest.mark.parametrize("name", ["img", "seg"])
def test_against_the_reference_fixture(fx, img_model, seg_model, name):
    c = fx[name]
    m = img_model if name == "img" else seg_model
    x = case_input(fx, name).to(DEV)
    z, _ = _eval_quantiser(m, x)
    tok = m.encode_code(x)
    e_z = sampled_err(z, c["latent"])
    assert e_z < 3e-3, e_z                                   # fp16-operand convolutions through 23 layers, as in test_gpu_parity
    E = m.quantize.embedding.weight.detach().cpu()
    zf = z.permute(0, 2, 3, 1).reshape(-1, E.shape[1]).cpu()
    mism = _explain_index_mismatches(zf, E, tok.flatten().cpu(), c["idx"].flatten())
    print("%s: latent error %.2e, %d of %d indices differ (each a boundary crossing of our latent)" % (name, e_z, mism, tok.numel()))
    assert mism <= 26, mism                                  # 5 % of the 512 rows
    dec = m.decode_code(c["idx"].to(DEV))
    e_d = sampled_err(dec.contiguous(), c["dec"])
    assert e_d < 5e-3, e_d


# ------------------------------------------------------------------------------------------------ no side effects
@pytest.mark.parametrize("q_counter", ["warm-up", "re-init"])
def test_train_mode_model_is_left_alone(img_model, q_counter):
    """A train-mode model at q_counter = 0 (Codebook.forward would return no indices) and one step before a k-means
    re-initialisation (it would replace the codebook), with a reservoir and deferred collection set, under enable_grad."""
    m = img_model
    x = _images(2, seed=5)
    want = _eval_quantiser(m, x)[1]
    cb = m.quantize
    m.train()
    saved = cb.q_counter, cb.reservoir
    cb.q_counter = 0 if q_counter == "warm-up" else cb.q_init - 1
    cb.reservoir = torch.randn(cb.q_init, cb.codebook_dim, device=DEV)
    cb.defer_collect = True
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    modes = {n: mod.training for n, mod in m.named_modules()}
    q, res, res_val = cb.q_counter, cb.reservoir, cb.reservoir.clone()
    try:
        with torch.enable_grad():
            tok = m.encode_code(x)
        assert torch.equal(tok.flatten(), want)
        assert not tok.requires_grad and tok.grad_fn is None
        now = m.state_dict()
        for k, v in sd.items():
            assert torch.equal(now[k], v), k                 # num_batches_tracked and the running statistics included
        assert {n: mod.training for n, mod in m.named_modules()} == modes
        assert cb.q_counter == q and cb.reservoir is res and torch.equal(cb.reservoir, res_val)
        assert not hasattr(cb, "_deferred_z") and cb.defer_collect is True
        assert all(p.grad is None for p in m.parameters())
    finally:
        del cb.defer_collect
        cb.q_counter, cb.reservoir = saved
        m.eval()


# ------------------------------------------------------------------------------------------------ validation
def test_validation(img_model, seg_model):
    from models import VQBASE
    x = _images(1, size=32)
    lab = torch.zeros(1, 4, 32, 32, dtype=torch.uint8, device=DEV)
    for m, bad in ((img_model, x.cpu()),                                  # a CPU tensor
                   (img_model, x.double()), (img_model, x.half()), (img_model, x.long()),   # dtypes
                   (img_model, lab), (img_model, torch.zeros(1, 4, 32, 32, device=DEV)),    # channel counts
                   (seg_model, lab[:, :3]), (seg_model, torch.zeros(1, 4, 32, 32, device=DEV)),
                   (seg_model, torch.zeros(1, 160, 32, 32, device=DEV)),
                   (img_model, _images(1, size=40)), (img_model, x[..., :24]), (seg_model, lab[..., :8, :])):  # H / W off 16
        with pytest.raises(ValueError):
            m.encode_code(bad)
    torch.manual_seed(0)
    cpu_model = VQBASE(TINY, 64, 32, 10, 100)                             # a CUDA tensor for a model on the CPU
    with pytest.raises(ValueError):
        cpu_model.encode_code(_images(1, size=16))


# ------------------------------------------------------------------------------------------------ the chain into MakeAScene
def test_tokens_feed_generate_score_and_decode_code():
    """Two small seeded VQ models whose 8 x 8 grids match a small seeded MakeAScene: compact scene planes -> seg_tokens,
    photo -> img_tokens; generate keeps given tokens (all, or those outside an edited box); score takes encode_code's tokens;
    decode_code turns a token grid back into an image."""
    from models import VQBASE
    from models.transformer import MakeAScene
    torch.manual_seed(0)
    vq_img = VQBASE(TINY, 96, 32, 10, 100).to(DEV)
    vq_seg = VQBASE(dict(TINY, in_channels=159, out_channels=159), 48, 32, 10, 100).to(DEV)
    for vq in (vq_img, vq_seg):
        with torch.no_grad():
            vq.quantize.embedding.weight.normal_()
    mas = MakeAScene(num_layers=2, hidden_dim=64, num_attn_heads=4, image_vocab_size=96, seg_vocab_size=48, text_vocab_size=92,
                     image_tokens_per_dim=8, seg_tokens_per_dim=8, text_length=12).to(DEV).eval()
    mas.device = DEV
    B = 3
    g = torch.Generator().manual_seed(9)
    lab = recipe.labels(1, n=B, size=16, cell=4).to(DEV)
    photo = (torch.rand(B, 3, 16, 16, generator=g) * 2 - 1).to(DEV)
    text = torch.randint(1, 80, (B, 12), generator=g).to(DEV)
    seg = vq_seg.encode_code(lab).flatten(1)
    img = vq_img.encode_code(photo).flatten(1)
    assert seg.shape == (B, 64) and img.shape == (B, 64) and int(seg.max()) < 48 and int(img.max()) < 96
    assert torch.equal(mas.generate(text, seg, img_tokens=img), img)
    region = torch.zeros(B, 16, 16, dtype=torch.bool, device=DEV)
    region[:, 3:11, 5:13] = True                                         # the edited box, in pixels
    keep = ~F.max_pool2d(region[:, None].float(), 2).bool().flatten(1)  # tokens whose 2 x 2 patch lies wholly outside it
    assert 0 < int(keep.sum()) < keep.numel()
    tok = mas.generate(text, seg, img_tokens=img, img_mask=keep, generator=torch.Generator(device=DEV).manual_seed(1))
    assert torch.equal(tok[keep], img[keep])
    lp = mas.score(text, seg, vq_img.encode_code(photo).flatten(1))
    assert lp.shape == (B, 64) and bool(torch.isfinite(lp).all()) and bool((lp <= 0).all())
    out = vq_img.decode_code(tok.view(B, 8, 8))
    assert out.shape == (B, 3, 16, 16)


# ------------------------------------------------------------------------------------------------ round trip
def test_round_trip_against_the_eval_forward(img_model):
    """decode_code(encode_code(x)) decodes the codebook rows e; the eval forward decodes the straight-through z + (e - z),
    which equals e up to fp32 rounding. Both decodes are measured against an fp64 decode of their own input (the oracle's
    restatement of the decoder, run in fp64); the tolerance is the fp64 effect of the rounding plus both measured kernel
    errors."""
    from oracle import vqgan_oracle as O
    m = img_model.eval()
    x = _images(1, seed=11)
    seen = {}
    hook = m.quantize.register_forward_hook(lambda _m, i, o: seen.update(z=i[0].detach(), zq=o[0].detach()))
    with torch.no_grad():
        dec = m(x)[0]
    hook.remove()
    tok = m.encode_code(x)
    rt = m.decode_code(tok)
    e = m.quantize.get_codebook_entry(tok.reshape(-1), (1, 16, 16, 256))
    zq = seen["zq"]
    z = seen["z"].double()
    d_in = float((zq.double() - e.double()).norm() / e.double().norm())
    # |fl(z + fl(e - z)) - e| <= u (|e - z| + |e|) (1 + u) element by element, u = 2^-24
    assert float((zq.double() - e.double()).norm()) <= 2.0 ** -24 * 1.001 * float((e.double() - z).norm() + e.double().norm())
    sd = {k: v.double() for k, v in m.state_dict().items()}
    with torch.no_grad():
        f = lambda q: O.run_plan(O.decoder_plan(**recipe.IMG), sd, "decoder.model", O.conv(q.double().contiguous(), sd, "post_quant_conv"))
        f_e, f_zq = f(e), f(zq)
    d64 = rel_err(f_zq, f_e)
    k_e, k_zq = rel_err(rt, f_e), rel_err(dec, f_zq)
    diff = rel_err(rt, dec)
    print("round trip: input %.2e, fp64 output %.2e, kernel errors %.2e / %.2e, rt vs forward %.2e" % (d_in, d64, k_e, k_zq, diff))
    assert k_e < 5e-3 and k_zq < 5e-3
    assert diff <= d64 + k_e + k_zq
