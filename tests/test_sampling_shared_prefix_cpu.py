"""MakeAScene.generate(num_samples=n), checked WITHOUT a GPU: the emulated C-ABI of tests/test_sampling_controls_cpu.py plus an
fp64 emulation of mas_attn_decode_shared_append(_f16) (include/mas_b200.h) that runs the unshared entry's emulation on the
concatenated cache. What is under test is the host side: n samples per prompt give the repeat_interleave call's tokens and
logits, the prefix pass runs once per prompt, the caches have the shared layout, and num_samples=1 changes nothing."""
import numpy as np
import pytest
import torch

from test_host_logic_cpu import Emu, _addr, _f32
from test_sampling_batched_cpu import BatchedEmu, _f16, _model, _tile
from test_sampling_controls_cpu import ControlsEmu

APPEND = ("mas_attn_decode_shared_append", "mas_attn_decode_shared_append_f16")
SHARED = APPEND + ("mas_attn_decode_shared", "mas_attn_decode_shared_f16")


class SharedEmu(ControlsEmu):
    """ControlsEmu + the shared-prefix decode attention: row r's cache is prefix row r // n followed by its suffix cache.
    `last` is the appended position (the _append entries) or the length (the others); either way the last position attended
    lies in the suffix."""

    def _shared(self, unshared, view, dt, qkv, kp, vp, ks, vs, ctx, R, n, heads, hd, P, Tsuf, last, rows_per_block):
        own = last if unshared in (Emu.mas_attn_decode_append, BatchedEmu.mas_attn_decode_append_f16) else last - 1
        assert R % n == 0 and P <= own < P + Tsuf and rows_per_block == 0
        Kp, Vp = (view(a, R // n * heads * P * hd).reshape(R // n, heads, P, hd) for a in (kp, vp))
        Ks, Vs = (view(a, R * heads * Tsuf * hd).reshape(R, heads, Tsuf, hd) for a in (ks, vs))
        K = torch.from_numpy(np.ascontiguousarray(np.concatenate([np.repeat(Kp, n, 0), Ks], 2))).to(dt)
        V = torch.from_numpy(np.ascontiguousarray(np.concatenate([np.repeat(Vp, n, 0), Vs], 2))).to(dt)
        unshared(self, qkv, K, V, ctx, R, heads, hd, P + Tsuf, last)
        Ks[...] = K[:, :, P:].numpy()
        Vs[...] = V[:, :, P:].numpy()

    def mas_attn_decode_shared_append(self, *a):
        self._shared(Emu.mas_attn_decode_append, lambda p, k: _f32(_addr(p), k), torch.float32, *a)

    def mas_attn_decode_shared_append_f16(self, *a):
        self._shared(BatchedEmu.mas_attn_decode_append_f16, lambda p, k: _f16(p, k), torch.float16, *a)

    def mas_attn_decode_shared(self, *a):
        self._shared(Emu.mas_attn_decode, lambda p, k: _f32(_addr(p), k), torch.float32, *a)

    def mas_attn_decode_shared_f16(self, *a):
        self._shared(BatchedEmu.mas_attn_decode_f16, lambda p, k: _f16(p, k), torch.float16, *a)


@pytest.fixture
def emu(monkeypatch):
    from mas_b200 import ops
    e = SharedEmu()
    monkeypatch.setattr(ops.L, "call", e)
    monkeypatch.setattr(ops, "_need_cuda", lambda x: None)
    monkeypatch.setattr(ops, "_tc_on", lambda: False)
    monkeypatch.setattr(ops.L, "query", lambda name, *a: 256)
    monkeypatch.setattr(torch.cuda, "graph_pool_handle", lambda: None)
    return e


def _inputs(B, sandwich=True):
    m, g = _model("tiny")
    if not sandwich:                        # the configuration of _decode_step_plain: residual adds without sandwich LayerNorm
        for layer in m.transformer.layers:
            layer.cogview_sandwich_layernorm = False
    return m, _tile(g["text"], B), _tile(g["seg"], B)


def _scalars(args):
    return [(name, [x for x in a if isinstance(x, (int, float))]) for name, a in args]


def test_num_samples_1_issues_the_same_entries(emu):
    """num_samples=1 passed explicitly issues the entries (with the same scalar arguments) of the call without it, and no
    shared-prefix entry, at fp32 and fp16 row counts, sampling and teacher-forced."""
    for B, kw in [(2, dict(temperature=0.9, top_k=20, generator="g")), (6, dict(guidance_scale=2.5, temperature=0.9, top_p=0.8,
                                                                                generator="g")), (2, dict(img_tokens="img"))]:
        m, text, seg = _inputs(B)
        runs = []
        for extra in ({}, {}, dict(num_samples=1)):                 # the first call builds the cached weight images
            k = dict(kw, **extra)
            if k.get("generator"):
                k["generator"] = torch.Generator().manual_seed(3)
            if k.get("img_tokens") is not None:
                k["img_tokens"] = _tile(_model("tiny")[1]["img"], B)
            emu.args.clear()
            toks = m.generate(text, seg, **k)
            runs.append((_scalars(emu.args), toks))
        assert runs[1][0] == runs[2][0] and torch.equal(runs[1][1], runs[2][1]), kw
        assert not [n for n, _ in runs[0][0] + runs[2][0] if n in SHARED]


CASES = [  # B, n, guidance scale, rows R (<= 8: fp32 decoding, above: fp16)
    (1, 4, 2.5, 8), (2, 3, None, 6), (2, 5, 2.5, 20), (3, 4, None, 12)]


@pytest.mark.parametrize("sandwich", [True, False])
@pytest.mark.parametrize("B,n,scale,R", CASES)
@pytest.mark.parametrize("mode", ["sample", "mask", "teacher"])
def test_matches_the_repeat_interleave_call(emu, sandwich, B, n, scale, R, mode):
    m, text, seg = _inputs(B, sandwich)
    L = m.image_length
    uncond = torch.randint(1, 40, text.shape, generator=torch.Generator().manual_seed(B)) if scale else None
    kw = dict(guidance_scale=scale, return_logits=True)
    if mode != "teacher":
        kw.update(temperature=0.8, top_k=40, top_p=0.9)
    if mode != "sample":
        kw["img_tokens"] = torch.randint(0, m.image_token_embedding.num_embeddings, (B * n, L), generator=torch.Generator().manual_seed(5))
    if mode == "mask":
        kw["img_mask"] = torch.rand(B * n, L, generator=torch.Generator().manual_seed(6)) < 0.4
    g1, g2 = torch.Generator().manual_seed(11), torch.Generator().manual_seed(11)
    emu.args.clear()
    t1, l1 = m.generate(text, seg, uncond_text_tokens=uncond, generator=g1, num_samples=n, **kw)
    shared = [(name, a) for name, a in emu.args if name in SHARED]
    assert len(shared) == len(m.transformer.layers) * (L - 1) and {a[7] for _, a in shared} == {n}
    # the fused step appends in the attention; the unfused one appends to the suffix cache, then attends (as it does at n = 1)
    assert {name in APPEND for name, _ in shared} == {sandwich}
    if not sandwich:
        appends = [a for name, a in emu.args if name in ("mas_kv_append", "mas_kv_append_f16")]
        assert [(a[1], a[7], a[8]) for a in appends[len(m.transformer.layers):]] == [
            (R, L, t) for t in range(L - 1) for _ in m.transformer.layers]
    def rep(t):
        return t.repeat_interleave(n, 0)
    t2, l2 = m.generate(rep(text), rep(seg), uncond_text_tokens=None if uncond is None else rep(uncond), generator=g2, **kw)
    assert t1.shape == (B * n, L) and l1.shape == (B * n, L, m.image_token_embedding.num_embeddings)
    assert torch.equal(t1, t2) and torch.equal(l1, l2)
    assert torch.equal(g1.get_state(), g2.get_state())
    if mode == "teacher":
        assert torch.equal(t1, kw["img_tokens"])


@pytest.mark.parametrize("B,n,scale,R", CASES)
def test_prefix_runs_once_per_prompt_and_caches_have_the_shared_layout(emu, B, n, scale, R):
    from models.transformer import _GraphedDecoder
    m, text, seg = _inputs(B)
    layers = m.transformer.layers
    heads, P, L = layers[0].attn.num_attn_heads, m.text_length + m.seg_length, m.image_length
    hd = m.hidden_dim // heads
    prompts = R // n
    m.generate(text, seg, guidance_scale=scale, temperature=0.9, num_samples=n, generator=torch.Generator().manual_seed(1))
    appends = [a for name, a in emu.args if name in ("mas_kv_append", "mas_kv_append_f16")]
    assert [(a[1], a[2], a[7], a[8]) for a in appends] == [(prompts, P, P, 0)] * len(layers)     # P rows, T = Tmax = prefix
    embeds = [a for name, a in emu.args if name == "mas_embed3_forward"]
    assert embeds[0][7] == prompts * m.text_length                                                  # the prefix embedding: P rows
    f16 = R > 8
    dec = _GraphedDecoder(m, R, torch.device("cpu"), n)
    el = 2 if f16 else 4
    for caches, shape in ((dec.kc, (prompts, heads, P, hd)), (dec.vc, (prompts, heads, P, hd)),
                          (dec.suffix[0], (R, heads, L, hd)), (dec.suffix[1], (R, heads, L, hd))):
        assert len(caches) == len(layers)
        for c in caches:
            assert tuple(c.shape) == shape and c.dtype == (torch.float16 if f16 else torch.float32)
    per_layer = sum(c.numel() * c.element_size() for c in (dec.kc[0], dec.vc[0], dec.suffix[0][0], dec.suffix[1][0]))
    assert per_layer == 2 * el * heads * hd * (prompts * P + R * L)
    one = _GraphedDecoder(m, R, torch.device("cpu"))
    assert one.suffix is None and tuple(one.kc[0].shape) == (R, heads, m.total_length, hd)


def test_argument_validation(emu):
    m, text, seg = _inputs(2)
    L = m.image_length
    for bad in (0, -1, True, False, 2.0, "2", None, np.int64(2)):
        with pytest.raises(ValueError):
            m.generate(text, seg, num_samples=bad)
    img = torch.zeros(2, L, dtype=torch.int64)
    for kw in (dict(img_tokens=img),                                                      # per prompt, not per output row
               dict(img_tokens=img, img_mask=torch.zeros(2, L, dtype=torch.bool)),
               dict(img_tokens=torch.zeros(6, L, dtype=torch.int64), img_mask=torch.zeros(2, L, dtype=torch.bool)),
               dict(img_tokens=torch.zeros(6, L - 1, dtype=torch.int64))):
        with pytest.raises(ValueError):
            m.generate(text, seg, num_samples=3, **kw)
    assert not [n for n in emu.names if n in SHARED or n.startswith("mas_sample")]


def test_shared_emulation_stores_this_token_in_the_suffix(emu):
    """The emulated entry itself: k / v of the token land at suffix slot pos - P, the prefix is untouched."""
    R, n, heads, hd, P, Tsuf = 4, 2, 2, 8, 5, 3
    H = heads * hd
    gen = torch.Generator().manual_seed(0)
    qkv = torch.randn(R, 3 * H, generator=gen)
    kp, vp = torch.randn(R // n, heads, P, hd, generator=gen), torch.randn(R // n, heads, P, hd, generator=gen)
    ks, vs = torch.zeros(R, heads, Tsuf, hd), torch.zeros(R, heads, Tsuf, hd)
    kp0 = kp.clone()
    ctx = torch.empty(R, H)
    emu("mas_attn_decode_shared_append", qkv, kp, vp, ks, vs, ctx, R, n, heads, hd, P, Tsuf, P + 1, 0)
    assert torch.equal(ks[:, :, 1], qkv[:, H:2 * H].view(R, heads, hd)) and torch.equal(vs[:, :, 1], qkv[:, 2 * H:].view(R, heads, hd))
    assert torch.equal(kp, kp0) and not ks[:, :, 0].any()
    q = qkv[:, :H].view(R, heads, 1, hd).double()
    K = torch.cat([kp.repeat_interleave(n, 0), ks[:, :, :2]], 2).double()
    V = torch.cat([vp.repeat_interleave(n, 0), vs[:, :, :2]], 2).double()
    ref = (torch.softmax(q @ K.transpose(-1, -2) / hd ** 0.5, -1) @ V).view(R, H)
    assert torch.allclose(ctx.double(), ref, atol=1e-6)
