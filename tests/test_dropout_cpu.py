"""Dropout of the token transformer without a GPU: a numpy restatement of the mask (Philox4x32-10, include/mas_b200.h) checked
against Random123's known-answer vectors, and the host logic of the dropout units and modules above the numpy C-ABI emulation
of test_host_logic_cpu, extended with the dropout entries. The whole tiny model with dropout is compared with the reference's
own models/transformer.py whose three nn.Dropout sites apply the same masks."""
import os

import numpy as np
import pytest
import torch

from test_host_logic_cpu import Emu, _addr, _f32, _i64, _tiny_model

M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Philox4x32-10 on uint64 arrays holding 32-bit words: ctr = 4 arrays, key = 2 arrays (broadcast)."""
    c = [np.asarray(v, dtype=np.uint64) for v in ctr]
    k0, k1 = (np.asarray(v, dtype=np.uint64) for v in key)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [((p1 >> np.uint64(32)) ^ c[1] ^ k0) & M32, p1 & M32, ((p0 >> np.uint64(32)) ^ c[3] ^ k1) & M32, p0 & M32]
        k0 = (k0 + np.uint64(0x9E3779B9)) & M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & M32
    return c


def keep_mask(seed, n, p):
    """keep(e) for e = 0 .. n-1 of a site with this int64 seed and probability p (bool array)."""
    s = int(seed) & 0xFFFFFFFFFFFFFFFF
    e = np.arange(n, dtype=np.uint64)
    g = e >> np.uint64(2)
    w = philox4x32_10([g & M32, g >> np.uint64(32), np.zeros_like(g), np.zeros_like(g)], [np.uint64(s & 0xFFFFFFFF), np.uint64(s >> 32)])
    word = np.choose((e & np.uint64(3)).astype(np.int64), w)
    return word >= np.uint64(int(np.floor(p * 2.0 ** 32)))


def scale_of(p):
    return 1.0 / (1.0 - p) if p < 1.0 else 0.0


def test_philox_known_answers():
    want = {((0, 0, 0, 0), (0, 0)): (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8),
            ((0xffffffff,) * 4, (0xffffffff,) * 2): (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd),
            ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0)): (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)}
    for (ctr, key), out in want.items():
        assert tuple(int(v) for v in philox4x32_10(ctr, key)) == out


def test_keep_rule_edges():
    for seed in (0, -1, 123456789012345):
        assert keep_mask(seed, 4099, 0.0).all()
        assert not keep_mask(seed, 4099, 1.0).any()
    m = keep_mask(7, 1 << 16, 0.25)
    assert abs(m.mean() - 0.75) < 0.01
    assert not np.array_equal(keep_mask(7, 256, 0.5), keep_mask(8, 256, 0.5))


class DropEmu(Emu):
    """Emu plus the dropout entries; records (entry, seed value) of every call that takes a seed."""

    def __init__(self):
        super().__init__()
        self.seeds = []

    def _seed(self, name, seed):
        v = int(_i64(_addr(seed), 1)[0])
        self.seeds.append((name, v))
        return v

    def mas_dropout(self, x, residual, y, n, p, scale, seed):
        k = keep_mask(self._seed("mas_dropout", seed), n, p)
        v = np.where(k, (_f32(_addr(x), n).astype(np.float64) if x is not None else 1.0) * scale, 0.0)
        if residual is not None:
            v = v + _f32(_addr(residual), n)
        _f32(_addr(y), n)[...] = v

    def mas_softmax_causal_dropout_backward(self, p, dp, ds, mats, rows, cols, scale, drop_p, seed):
        n = mats * rows * cols
        k = keep_mask(self._seed("mas_softmax_causal_dropout_backward", seed), n, drop_p).reshape(mats, rows, cols)
        P = _f32(_addr(p), n).reshape(mats, rows, cols).astype(np.float64)
        dP = _f32(_addr(dp), n).reshape(mats, rows, cols).astype(np.float64)
        vis = np.tril(np.ones((rows, cols)), cols - rows) > 0
        g = np.where(vis & k, dP * scale_of(drop_p), 0.0)
        _f32(_addr(ds), n).reshape(mats, rows, cols)[...] = np.where(vis, P * (g - (g * P).sum(-1, keepdims=True)) * scale, 0.0)

    def _dropped(self, name, a, R, H, p, seed):
        k = keep_mask(self._seed(name, seed), R * H, p).reshape(R, H)
        return np.where(k, _f32(_addr(a), R * H).reshape(R, H).astype(np.float64) * scale_of(p), 0.0), k

    def mas_layernorm_dropout_forward(self, a, gamma, beta, residual, y, mean, rstd, R, H, eps, p, seed):
        X, _ = self._dropped("mas_layernorm_dropout_forward", a, R, H, p, seed)
        m = X.mean(-1)
        rs = 1.0 / np.sqrt(((X - m[:, None]) ** 2).mean(-1) + eps)
        o = (X - m[:, None]) * rs[:, None] * _f32(_addr(gamma), H) + _f32(_addr(beta), H)
        if residual is not None:
            o = o + _f32(_addr(residual), R * H).reshape(R, H)
        _f32(_addr(y), R * H).reshape(R, H)[...] = o
        _f32(_addr(mean), R)[...] = m
        _f32(_addr(rstd), R)[...] = rs

    def mas_layernorm_dropout_backward(self, dy, a, mean, rstd, gamma, da, dgamma, dbeta, R, H, p, seed, ws, ws_bytes):
        X, k = self._dropped("mas_layernorm_dropout_backward", a, R, H, p, seed)
        D = _f32(_addr(dy), R * H).reshape(R, H).astype(np.float64)
        rs = _f32(_addr(rstd), R).astype(np.float64)[:, None]
        xh = (X - _f32(_addr(mean), R).astype(np.float64)[:, None]) * rs
        g = D * _f32(_addr(gamma), H)
        dx = rs * (g - g.mean(-1, keepdims=True) - xh * (g * xh).mean(-1, keepdims=True))
        _f32(_addr(da), R * H).reshape(R, H)[...] = np.where(k, dx * scale_of(p), 0.0)
        _f32(_addr(dgamma), H)[...] = (D * xh).sum(0)
        _f32(_addr(dbeta), H)[...] = D.sum(0)


@pytest.fixture
def demu(monkeypatch):
    from mas_b200 import ops
    e = DropEmu()
    monkeypatch.setattr(ops.L, "call", e)
    monkeypatch.setattr(ops, "_need_cuda", lambda x: None)
    monkeypatch.setattr(ops, "_tc_on", lambda: False)
    monkeypatch.setattr(ops.L, "query", lambda name, *a: 256)
    drawn = []
    orig = ops.dropout_seed

    def record(device):
        s = orig(device)
        drawn.append(int(s[0]))
        return s
    monkeypatch.setattr(ops, "dropout_seed", record)
    e.drawn = drawn
    return e


def _dropout_model(p_attn, p_out, sandwich=True):
    from models.transformer import MakeAScene
    m, g = _tiny_model()
    d = MakeAScene(**g["cfg"], attn_dropout_prob=p_attn, out_dropout_prob=p_out)
    if not sandwich:
        for l in d.transformer.layers:
            l.cogview_sandwich_layernorm = False
    d.load_state_dict(g["state_dict"])
    d.device = torch.device("cpu")
    return d, g


def _step(m, g):
    m.zero_grad()
    loss = m.loss(g["text"], g["seg"], g["img"])
    loss.backward()
    return loss


def test_each_site_has_one_seed_per_call_shared_by_its_backward(demu):
    torch.manual_seed(0)
    m, g = _dropout_model(0.2, 0.3)
    _step(m, g)
    _step(m, g)
    layers = len(m.transformer.layers)
    assert len(demu.drawn) == 2 * 3 * layers                          # 3 sites per layer and step
    assert len(set(demu.drawn)) == len(demu.drawn)                    # sites, layers and steps all differ
    by_seed = {}
    for name, s in demu.seeds:
        by_seed.setdefault(s, []).append(name)
    assert set(by_seed) == set(demu.drawn)
    for s, names in by_seed.items():
        if "mas_layernorm_dropout_forward" in names:
            assert names == ["mas_layernorm_dropout_forward", "mas_layernorm_dropout_backward"]
        else:   # attention, fallback path: forward staging of P * keep, backward staging and the softmax backward
            assert names == ["mas_dropout", "mas_dropout", "mas_softmax_causal_dropout_backward"]


def test_zero_probability_and_eval_mode_launch_todays_entries(demu):
    torch.manual_seed(0)
    ref, g = _tiny_model()
    _step(ref, g)
    today = list(demu.names)
    assert not demu.drawn
    for p_attn, p_out, train in ((0.0, 0.0, True), (0.1, 0.1, False), (0.5, 0.0, False)):
        demu.names.clear()
        m, _ = _dropout_model(p_attn, p_out)
        m.train(train)
        _step(m, g)
        assert demu.names == today and not demu.drawn
    # generate() never draws a mask, in train mode either
    m, _ = _dropout_model(0.3, 0.3)
    m.train()
    with torch.no_grad():
        m.generate(g["text"], g["seg"], img_tokens=g["img"])
    assert not demu.drawn


def _reference_with_masks(g, seeds, p_attn, p_out, sandwich):
    """The staged reference MakeAScene with its three nn.Dropout modules per layer replaced by ones applying the masks of the
    recorded seeds (in forward order: attention, out_drop, mlp.dropout of each layer - the order the drop-in draws them)."""
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
    try:
        import vendor_ref
    finally:
        sys.path.pop(0)
    if not vendor_ref.available():
        pytest.skip("the reference's model files are not staged under oracle/_ref")
    import importlib
    vendor_ref.load_models()
    R = importlib.import_module("_mas_ref_models.transformer")
    ref = R.MakeAScene(**g["cfg"]).double()
    ref.load_state_dict(g["state_dict"])
    ref.device = torch.device("cpu")
    queue = list(seeds)

    class Masked(torch.nn.Module):
        def __init__(self, p):
            super().__init__()
            self.p = p

        def forward(self, x):
            if self.p == 0:     # the drop-in draws no seed for a site at p = 0
                return x
            k = keep_mask(queue.pop(0), x.numel(), self.p).reshape(x.shape)
            return x * torch.from_numpy(k).to(x.dtype) * scale_of(self.p)
    for l in ref.transformer.layers:
        l.attn.attn_drop, l.attn.out_drop, l.mlp.dropout = Masked(p_attn), Masked(p_out), Masked(p_out)
        l.cogview_sandwich_layernorm = sandwich
    return ref, queue


@pytest.mark.parametrize("p_attn,p_out,sandwich", [(0.2, 0.3, True), (0.5, 0.1, False), (1.0, 0.0, True), (0.0, 1.0, True)])
def test_tiny_model_with_dropout_matches_reference_under_the_same_masks(demu, p_attn, p_out, sandwich):
    from conftest import rel_err
    torch.manual_seed(3)
    m, g = _dropout_model(p_attn, p_out, sandwich)
    loss = _step(m, g)
    ref, queue = _reference_with_masks(g, demu.drawn, p_attn, p_out, sandwich)
    logits = ref(g["text"], g["seg"], g["img"])
    rl = torch.nn.functional.cross_entropy(logits.reshape(-1, logits.shape[-1]), g["img"].reshape(-1))
    rl.backward()
    assert not queue
    assert abs(float(loss.detach()) - float(rl)) < 1e-5 * max(1.0, float(rl))
    rnamed = dict(ref.named_parameters())
    for k, p in m.named_parameters():
        if p.grad is None:      # the unused sandwich LayerNorms without sandwich_layernorm
            assert rnamed[k].grad is None, k
        else:
            assert rel_err(p.grad, rnamed[k].grad) < 1e-4, k


def test_module_units_apply_their_own_dropout(demu):
    """SelfAttention / MLP called on their own drop their output like the reference's modules; eval mode is the identity."""
    from models.transformer import MLP
    torch.manual_seed(1)
    mlp = MLP(8, 0.4)
    x = torch.randn(3, 5, 8)
    y = mlp(x)
    base = mlp.project(x).detach()
    k = keep_mask(demu.drawn[0], x.numel(), 0.4).reshape(base.shape)
    assert torch.allclose(y.detach().double(), torch.where(torch.from_numpy(k), base.double() / 0.6, 0.0), atol=1e-6)
    mlp.eval()
    assert torch.equal(mlp(x).detach(), base)


def test_probability_validation(demu):
    from models.transformer import MakeAScene, MLP, SelfAttention, Transformer, TransformerLayer
    for bad in (-0.1, 1.5):
        with pytest.raises(ValueError):
            SelfAttention(8, 2, bad, 0.0)
        with pytest.raises(ValueError):
            SelfAttention(8, 2, 0.0, bad)
        with pytest.raises(ValueError):
            MLP(8, bad)
        with pytest.raises(ValueError):
            TransformerLayer(8, 2, bad, 0.0)
        with pytest.raises(ValueError):
            Transformer(1, 8, 2, 2, 2, 4, attn_dropout_prop=bad)
        with pytest.raises(ValueError):
            MakeAScene(1, 8, 2, 16, 16, 16, 2, 2, 4, out_dropout_prob=bad)
    m = MLP(8, 0.1)
    m.dropout.p = 1.5
    with pytest.raises(ValueError):
        m(torch.zeros(2, 8))
    with pytest.raises(NotImplementedError):
        SelfAttention(8, 2, 0.1, 0.1, rudalle_relax=True)
    with pytest.raises(NotImplementedError):
        TransformerLayer(8, 2, 0.1, 0.1, cogview_layernorm_prescale=True)
