"""CPU: the oracle restatement (oracle/vqgan_oracle.py) is pinned against fixtures produced by the
REAL reference (oracle/make_golden.py). No GPU, no product code."""
import os

import numpy as np
import torch

from conftest import GOLDEN, rel_err
from oracle import vqgan_oracle as O


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def test_tiny_vqbase_forward_backward_matches_reference():
    g = _load("vqbase_tiny.pt")
    sd = {k: v.clone().requires_grad_(k in g["grads"]) for k, v in g["state_dict"].items()}
    taps = {}
    dec, diff, idx = O.vqbase_forward(sd, g["ddconfig"], g["x"], taps=taps)
    assert torch.equal(idx, g["idx"])
    assert rel_err(dec, g["dec"]) < 1e-5
    assert abs(float(diff) - float(g["diff"])) < 1e-6
    for k, v in g["taps"].items():
        assert rel_err(taps[k], v) < 1e-5, k
    loss = O.proxy_loss(g["x"], dec, diff)
    loss.backward()
    for k, gv in g["grads"].items():
        assert rel_err(sd[k].grad, gv) < 2e-4, k


def test_tiny_modes_bypass_and_eval():
    g = _load("vqbase_tiny.pt")
    m = _load("vqbase_tiny_modes.pt")
    dec, diff, idx = O.vqbase_forward(g["state_dict"], g["ddconfig"], g["x"], quantize=False, training=True)
    assert idx is None and float(diff) == 0.0
    assert rel_err(dec, m["dec_bypass"]) < 1e-5
    dec, diff, idx = O.vqbase_forward(g["state_dict"], g["ddconfig"], g["x"], quantize=True, training=False)
    assert rel_err(dec, m["dec_eval"]) < 1e-5
    assert abs(float(diff) - float(m["diff_eval"])) < 1e-6


def test_codebook_sets():
    sets = _load("codebook_sets.pt")
    for name, s in sets.items():
        z = s["z"].clone().requires_grad_(True)
        E = s["E"].clone().requires_grad_(True)
        z_q, loss, idx = O.codebook_forward(z, E)
        assert torch.equal(idx, s["idx"]), name
        assert torch.allclose(z_q, s["z_q"], atol=1e-6), name
        assert abs(float(loss) - float(s["loss"])) < 1e-6 * max(1.0, abs(float(s["loss"]))), name
        (z_q * torch.linspace(-1, 1, z_q.numel()).view_as(z_q)).sum().add(loss).backward()
        assert rel_err(z.grad, s["grad_z"]) < 1e-5, name
        assert rel_err(E.grad, s["grad_E"]) < 1e-5, name
        assert torch.equal(O.codebook_entry(s["E"], s["idx"], (3, 4, 4, 64)), s["entry"])
        # numpy restatement of the integer-valued argmin: identical except on exact-tie sets
        zf = s["z"].permute(0, 2, 3, 1).reshape(-1, 64).numpy()
        idx_np = O.codebook_argmin_numpy(zf, s["E"].numpy())
        bad = np.nonzero(idx_np != s["idx"].numpy())[0]
        if name in ("trained", "clustered"):
            assert bad.size == 0, name
        else:
            gap, ulp = O.codebook_gap_fp64(torch.from_numpy(zf), s["E"], torch.from_numpy(idx_np), s["idx"])
            assert bool((gap[bad] <= 4 * ulp[bad]).all()), name


def test_blocks():
    blocks = _load("blocks.pt")
    fn = {"res": O.resnet_block, "attn": O.attn_block, "down": O.downsample, "up": O.upsample}
    for name, b in blocks.items():
        sd = {"m." + k: v.clone().requires_grad_(True) for k, v in b["state_dict"].items()}
        x = b["x"].clone().requires_grad_(True)
        y = fn[name.split("_")[0]](x, sd, "m")
        assert rel_err(y, b["y"]) < 1e-5, name
        (y * torch.linspace(-1, 1, y.numel()).view_as(y)).sum().backward()
        assert rel_err(x.grad, b["grad_x"]) < 1e-4, name
        for k, gv in b["grads"].items():
            assert rel_err(sd["m." + k].grad, gv) < 1e-4, (name, k)


def _sampled_err(t, fx, norm):
    """Fixture entries stored as (strided sample, stride): error of the same sample, relative to the full tensor's
    norm scaled to the sample size."""
    smp, stride = fx
    got = t.detach().reshape(-1)[::stride].double().cpu()
    scale = norm * (smp.numel() / t.numel()) ** 0.5
    return float((got - smp.double()).norm() / max(scale, 1e-30))


def build_tc_block(name, M):
    import torch.nn as nn
    kind = {"res_128_128": lambda: M.ResnetBlock(in_channels=128, out_channels=128, dropout=0.0),
            "res_128_256": lambda: M.ResnetBlock(in_channels=128, out_channels=256, dropout=0.0),
            "res_512_512": lambda: M.ResnetBlock(in_channels=512, out_channels=512, dropout=0.0),
            "attn_512": lambda: M.AttnBlock(512),
            "attn_res_512": lambda: nn.Sequential(M.AttnBlock(512), M.ResnetBlock(in_channels=512, out_channels=512, dropout=0.0)),
            "res_res_attn_512": lambda: nn.Sequential(M.ResnetBlock(in_channels=512, out_channels=512, dropout=0.0),
                                                      M.ResnetBlock(in_channels=512, out_channels=512, dropout=0.0), M.AttnBlock(512)),
            "up_128": lambda: M.Upsample(128, True), "down_128": lambda: M.Downsample(128, True),
            "up_512": lambda: M.Upsample(512, True)}
    return kind[name]()


def _oracle_tc_block(name, x, sd):
    if name == "attn_res_512":
        return O.resnet_block(O.attn_block(x, sd, "m.0"), sd, "m.1")
    if name == "res_res_attn_512":
        return O.attn_block(O.resnet_block(O.resnet_block(x, sd, "m.0"), sd, "m.1"), sd, "m.2")
    fn = {"res": O.resnet_block, "attn": O.attn_block, "down": O.downsample, "up": O.upsample}
    return fn[name.split("_")[0]](x, sd, "m")


def test_tensor_path_blocks_oracle_matches_reference():
    """blocks_tc.pt (wide blocks the tensor-core kernels take; weights regenerated from seeds, oracle/seeded.py): the
    restatement agrees with the REAL reference's outputs and gradients. The drop-in modules are used on the CPU as
    parameter holders only (no kernel runs): their parameter names / shapes are the reference's."""
    from models import modules as M
    from oracle.seeded import assert_same_fill, fill_seeded, seeded_input
    blocks = _load("blocks_tc.pt")
    for name, b in blocks.items():
        mod = build_tc_block(name, M)
        assert_same_fill(fill_seeded(mod, b["seed_w"]), b["param_checks"])   # same names, order and values as on the reference
        sd = {"m." + k: v.detach().clone().requires_grad_(True) for k, v in mod.state_dict().items()}
        x = seeded_input(b["shape"], b["seed_x"], 1.5, 0.3).requires_grad_(True)
        y = _oracle_tc_block(name, x, sd)
        assert _sampled_err(y, b["y"], b["y_norm"]) < 1e-5, name
        (y * torch.linspace(-1, 1, y.numel()).view_as(y)).sum().backward()
        assert _sampled_err(x.grad, b["grad_x"], b["grad_x_norm"]) < 1e-4, name
        for k, gv in b["grads"].items():
            g = sd["m." + k].grad
            if k.endswith("k.bias"):
                continue                                   # mathematically zero (softmax shift invariance)
            e = _sampled_err(g, gv, b["grad_norms"][k]) if isinstance(gv, tuple) else rel_err(g, gv)
            assert e < 2e-4, (name, k, e)


def test_img_config_256_oracle_matches_reference():
    """vqbase_img_256.pt: the 95 M-parameter img_config model at BASELINE's 256x256 (batch 2), forward + backward."""
    from models import VQBASE
    g = _load("vqbase_img_256.pt")
    torch.manual_seed(0)
    m = VQBASE(g["ddconfig"], 8192, 256, 3000, 12500)      # CPU parameter holder: init is bit-identical (test_abi.py)
    with torch.no_grad():
        m.quantize.embedding.weight.normal_()
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    params = {k: v.requires_grad_(True) for k, v in sd.items() if v.is_floating_point() and "running" not in k}
    sd.update(params)
    x = torch.rand(g["x_shape"], generator=torch.Generator().manual_seed(g["x_seed"]))
    assert abs(float(x.double().sum()) - g["x_sum"]) < 1e-6
    taps = {}
    dec, diff, idx = O.vqbase_forward(sd, g["ddconfig"], x, taps=taps)
    assert torch.equal(idx, g["idx"])
    assert rel_err(taps["quant_conv"], g["quant_in"]) < 1e-5
    assert _sampled_err(dec, g["dec_sample"], g["dec_norm"]) < 1e-5
    assert abs(float(diff) - float(g["diff"])) < 1e-6
    O.proxy_loss(x, dec, diff).backward()
    for k, v in g["grad_norms"].items():
        assert _sampled_err(params[k].grad, g["grad_samples"][k], max(v, 1e-12)) < 5e-4 or v < 1e-7, k


def test_plans_match_img_config_layer_counts():
    g = _load("vqbase_img_64.pt")
    enc = O.encoder_plan(**g["ddconfig"])
    dec = O.decoder_plan(**g["ddconfig"])
    assert len(enc) == 23 and len(dec) == 29          # SURVEY.md 3.2
    assert sum(k == "attn" for k, *_ in enc) == 3 and sum(k == "attn" for k, *_ in dec) == 4


def test_seg_loss():
    g = _load("seg_loss.pt")
    pred = g["pred"].clone().requires_grad_(True)
    loss = O.bce_loss_with_quant(g["qloss"], g["target"], pred)
    assert abs(float(loss) - float(g["loss"])) < 1e-6
    loss.backward()
    assert rel_err(pred.grad, g["grad"]) < 1e-6


def test_transformer_oracle_matches_reference():
    from oracle import transformer_oracle as T
    for tag in ("tiny", "wide"):
        g = _load(f"transformer_{tag}.pt")
        sd = {k: v.clone().requires_grad_(k in g["grad_norms"]) for k, v in g["state_dict"].items()}
        logits = T.make_a_scene_forward(sd, g["cfg"], g["text"], g["seg"], g["img"])
        assert logits.shape == g["logits"].shape
        assert rel_err(logits, g["logits"]) < 1e-5, tag
        loss = torch.nn.functional.cross_entropy(logits.reshape(-1, logits.shape[-1]), g["img"].reshape(-1))
        assert abs(float(loss) - float(g["loss"])) < 1e-5
        loss.backward()
        for k, gv in g["grads"].items():
            assert rel_err(sd[k].grad, gv) < 2e-4, (tag, k)


def test_cached_sampling_oracle_matches_reference_logits():
    """oracle/transformer_oracle.generate_logits (KV-cached decoding, the algorithm MakeAScene.generate runs on the GPU):
    teacher-forced it reproduces the logits of the REAL reference's non-cached forward (fixture), and guided greedy
    decoding follows the arg-max of the mixed cond / uncond logits of two non-cached passes."""
    from oracle import transformer_oracle as T
    for tag in ("tiny", "wide"):
        g = _load(f"transformer_{tag}.pt")
        sd = {k: v.clone() for k, v in g["state_dict"].items()}
        with torch.no_grad():
            toks, lg = T.generate_logits(sd, g["cfg"], g["text"], g["seg"], img_tokens=g["img"])
        assert torch.equal(toks, g["img"])
        assert rel_err(lg, g["logits"]) < 1e-4
    g = _load("transformer_tiny.pt")
    sd = {k: v.clone() for k, v in g["state_dict"].items()}
    with torch.no_grad():
        toks, lg = T.generate_logits(sd, g["cfg"], g["text"], g["seg"], guidance_scale=2.5)
        cond = T.make_a_scene_forward(sd, g["cfg"], g["text"], g["seg"], toks)
        unc = T.make_a_scene_forward(sd, g["cfg"], torch.zeros_like(g["text"]), g["seg"], toks)
    assert rel_err(lg, unc + 2.5 * (cond - unc)) < 1e-4
    assert torch.equal(toks, lg.argmax(-1))
