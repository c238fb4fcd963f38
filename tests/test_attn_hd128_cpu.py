"""CPU: the routes of the 128-wide-head causal attention above the C-ABI (ops.L.call recorded, nothing launched): head dim
128 with S % 128 == 0 reaches the fused entries (stored P, P-free forward, recomputing backward) with hd = 128; other shapes
still raise before any call; MAS_ATTN_FUSED=0 keeps the GEMM / softmax / GEMM sequence."""
import pytest
import torch


@pytest.fixture
def calls(monkeypatch):
    from mas_b200 import ops
    rec = []
    monkeypatch.setattr(ops, "_need_cuda", lambda x: None)
    monkeypatch.setattr(ops, "_tc_on", lambda: True)
    monkeypatch.setattr(ops.L, "call", lambda *a: rec.append(a))
    monkeypatch.delenv("MAS_ATTN_FUSED", raising=False)
    return rec


def _names(rec):
    return [a[0] for a in rec]


def _entry(rec, name):
    got = [a for a in rec if a[0] == name]
    assert len(got) == 1, _names(rec)
    return got[0]


@pytest.mark.parametrize("S,heads", [(128, 1), (256, 2), (1408, 16)])
def test_recompute_reaches_the_fused_entries_with_hd128(S, heads, calls):
    from mas_b200 import ops
    qkv = torch.zeros(1, S, 3 * heads * 128, requires_grad=True)
    y = ops.CausalAttentionFn.apply(qkv, heads, 0.0, True)
    # mas_attn_causal_forward_stats(qkv, amax, stats, ctx, B, S, heads, hd, scale, p, seed)
    f = _entry(calls, "mas_attn_causal_forward_stats")
    assert f[6:10] == (S, heads, 128, 1.0 / 128 ** 0.5)
    assert tuple(f[3].shape) == (2, 1, heads, S)
    y.backward(torch.ones_like(y))
    # mas_attn_causal_backward(qkv, ctx, dctx, stats, amax, dctx_amax, D, dqkv, B, S, heads, hd, scale, p, seed)
    b = _entry(calls, "mas_attn_causal_backward")
    assert b[10:14] == (S, heads, 128, 1.0 / 128 ** 0.5)
    assert not any(n.startswith(("mas_gemm", "mas_softmax")) for n in _names(calls)), _names(calls)


@pytest.mark.parametrize("p", [0.0, 0.2])
def test_stored_p_reaches_the_fused_forward_with_hd128(p, calls, monkeypatch):
    from mas_b200 import ops
    monkeypatch.setattr(ops, "dropout_seed", lambda device: torch.zeros(1, dtype=torch.int64))
    qkv = torch.zeros(2, 256, 3 * 2 * 128)
    ops.CausalAttentionFn.apply(qkv, 2, p, False)
    f = _entry(calls, "mas_attn_causal_dropout_forward" if p > 0 else "mas_attn_causal_forward")
    assert f[6:9] == (256, 2, 128)
    assert not any(n.startswith(("mas_gemm", "mas_softmax")) for n in _names(calls)), _names(calls)


@pytest.mark.parametrize("S,hd", [(256, 32), (200, 64), (200, 128), (256, 96), (64, 128)])
def test_other_shapes_still_raise_before_any_call(S, hd, calls):
    from mas_b200 import ops
    qkv = torch.zeros(1, S, 3 * 2 * hd)
    with pytest.raises(RuntimeError, match="head dim 64, S % 128 == 0"):
        ops.CausalAttentionFn.apply(qkv, 2, 0.0, True)
    assert not calls
    assert not ops.attn_causal_fused_on(S, hd)


def test_fused_off_keeps_the_gemm_sequence_at_hd128(calls, monkeypatch):
    from mas_b200 import ops
    assert ops.attn_causal_fused_on(256, 128)
    monkeypatch.setenv("MAS_ATTN_FUSED", "0")
    assert not ops.attn_causal_fused_on(256, 128)
    qkv = torch.zeros(1, 256, 3 * 2 * 128)
    ops.CausalAttentionFn.apply(qkv, 2, 0.0, False)
    names = _names(calls)
    assert "mas_softmax_causal_forward" in names and names.count("mas_gemm_batched2") == 2, names
    assert not any(n.startswith("mas_attn_causal") for n in names), names
    with pytest.raises(RuntimeError, match="head dim 64, S % 128 == 0"):
        ops.CausalAttentionFn.apply(qkv, 2, 0.0, True)


def test_launch_trace_records_nothing_without_launches():
    """The launch trace the GPU tests assert their routes with: empty when nothing ran, off again after the block."""
    from mas_b200 import _lib
    with _lib.launch_trace() as names:
        pass
    assert names == []
    assert _lib.load().mas_launch_trace_read(None, 0) == 0
