"""Compact scene maps on the CPU: mas_b200.scene.pack (the host-side entry of untrusted label data) against a restatement of
the reference's PreprocessedDataset.load_segmentation (Data/dataset_preprocessor.py:61-86), and the host logic of the
compact VQ-SEG step (Conv3x3Fn / BCELogitsFn taking uint8 labels) above the emulated C-ABI of tests/test_host_logic_vq_cpu.py
with numpy restatements of mas_scene_expand and mas_bce_scene_*.  The kernels are tested on the GPU
(tests/test_gpu_scene_maps.py)."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from test_host_logic_vq_cpu import VQSEG_DD, VqEmu, _addr, _f32, _view4, _vqseg_model, vq_emu  # noqa: F401  (vq_emu: fixture)


def _u8(p, n):
    return np.ctypeslib.as_array((ctypes.c_uint8 * int(n)).from_address(_addr(p)))


def load_segmentation(seg_panoptic, seg_human, seg_face, edges_panoptic, edges_human):
    """Data/dataset_preprocessor.py:61-86 on in-memory arrays of one image -> [H, W, 159] float32."""
    pan = F.one_hot(torch.from_numpy(seg_panoptic + 1).to(torch.long), num_classes=134)[..., 1:]
    hum = F.one_hot(torch.from_numpy(seg_human + 1).to(torch.long), num_classes=21)[..., 1:]
    edges = (torch.from_numpy(edges_panoptic).unsqueeze(-1) + torch.from_numpy(edges_human).unsqueeze(-1)).float()
    face = F.one_hot(torch.from_numpy(seg_face).to(torch.long), num_classes=6)[..., 1:]
    return torch.cat([pan, hum, face, edges], dim=-1)


def expand_np(lab, c=159):
    """Documented semantics of mas_scene_expand (include/mas_b200.h): [N, 4, H, W] codes -> [N, H, W, c] map."""
    lab = lab.astype(np.int64)
    out = np.zeros(lab.shape[:1] + lab.shape[2:] + (c,), dtype=np.float32)
    for plane, base, k in ((0, 0, 133), (1, 133, 20), (2, 153, 5)):
        out[..., base:base + k] = lab[:, plane, :, :, None] == np.arange(1, k + 1)
    out[..., 158] = np.where(lab[:, 3] <= 2, lab[:, 3], 0)
    return out


def _random_arrays(rng, shape):
    return (rng.integers(-1, 133, shape), rng.integers(-1, 20, shape), rng.integers(0, 6, shape),
            rng.integers(0, 2, shape).astype(np.uint8), rng.integers(0, 2, shape).astype(np.uint8))


def test_pack_round_trips_and_expands_to_load_segmentation():
    from mas_b200 import scene
    rng = np.random.default_rng(0)
    pan, hum, face, ep, eh = _random_arrays(rng, (3, 9, 13))
    pan[0, 0, :3], hum[0, 0, :3], face[0, 0, :3] = (-1, 0, 132), (-1, 0, 19), (0, 1, 5)   # both ends of every range
    ep[0, 0, 0] = eh[0, 0, 0] = 1                                                         # edges = 2
    lab = scene.pack(pan, hum, face, ep + eh)
    assert lab.dtype == torch.uint8 and lab.shape == (3, 4, 9, 13) and lab.is_contiguous()
    assert np.array_equal(lab[:, 0].numpy().astype(np.int64) - 1, pan) and np.array_equal(lab[:, 1].numpy().astype(np.int64) - 1, hum)
    assert np.array_equal(lab[:, 2].numpy(), face) and np.array_equal(lab[:, 3].numpy(), ep + eh)
    dense = expand_np(lab.numpy())
    for i in range(3):
        ref = load_segmentation(pan[i], hum[i], face[i], ep[i], eh[i])
        assert torch.equal(torch.from_numpy(dense[i]), ref)
    one = scene.pack(torch.from_numpy(pan[1]), torch.from_numpy(hum[1]), torch.from_numpy(face[1]), torch.from_numpy(ep[1] + eh[1]))
    assert torch.equal(one, lab[1])                                       # one image, torch inputs
    assert torch.equal(scene.pack(pan[1], hum[1], face[1], (ep[1] + eh[1]).astype(bool)),
                       scene.pack(pan[1], hum[1], face[1], np.minimum(ep[1] + eh[1], 1)))   # bool edge maps


@pytest.mark.parametrize("plane,value", [(0, -2), (0, 133), (1, -2), (1, 20), (2, -1), (2, 6), (3, -1), (3, 3)])
def test_pack_rejects_out_of_range_codes(plane, value):
    from mas_b200 import scene
    arrays = [a.astype(np.int64) for a in _random_arrays(np.random.default_rng(1), (4, 5))[:3]] + [np.zeros((4, 5), np.int64)]
    arrays[plane][2, 3] = value
    with pytest.raises(ValueError):
        scene.pack(*arrays)


def test_pack_rejects_bad_dtypes_and_shapes():
    from mas_b200 import scene
    z = np.zeros((4, 5), np.int64)
    with pytest.raises(ValueError):
        scene.pack(z.astype(np.float32), z, z, z)
    with pytest.raises(ValueError):
        scene.pack(z, z, z, torch.zeros(4, 5))
    with pytest.raises(ValueError):
        scene.pack(z, z[:, :4], z, z)
    with pytest.raises(ValueError):
        scene.pack(z[0], z[0], z[0], z[0])                               # 1-D
    with pytest.raises(ValueError):
        scene.pack(z[None, None], z[None, None], z[None, None], z[None, None])   # 4-D
    with pytest.raises(ValueError):
        scene.pack(z[:0], z[:0], z[:0], z[:0])                            # empty


class SceneEmu(VqEmu):
    """VqEmu plus the compact scene-map entries."""

    def mas_scene_expand(self, labels, N, H, W, y, ys):
        assert (ys.n, ys.h, ys.w) == (N, H, W) and ys.c >= 159
        _view4(y, ys)[...] = expand_np(_u8(labels, N * 4 * H * W).reshape(N, 4, H, W), ys.c)

    def _dense_target(self, labels, N, H, W):
        return torch.from_numpy(expand_np(_u8(labels, N * 4 * H * W).reshape(N, 4, H, W)).transpose(0, 3, 1, 2).copy())

    def mas_bce_scene_forward(self, logits, labels, pos_weight, N, CP, H, W, loss_out, ws, ws_bytes):
        self.mas_bce_cl_forward(logits, self._dense_target(labels, N, H, W), pos_weight, N, 159, CP, H, W, loss_out, ws, ws_bytes)

    def mas_bce_scene_backward(self, logits, labels, pos_weight, g, N, CP, H, W, grad):
        self.mas_bce_cl_backward(logits, self._dense_target(labels, N, H, W), pos_weight, g, N, 159, CP, H, W, grad)


@pytest.fixture
def scene_emu(vq_emu, monkeypatch):  # noqa: F811
    from mas_b200 import ops
    e = SceneEmu()
    monkeypatch.setattr(ops.L, "call", e)
    monkeypatch.setattr(ops, "_need_cuda", lambda x, dtype=None: None)
    return e


def _labels(n=2, h=64, w=64, seed=5):
    g = torch.Generator().manual_seed(seed)
    return torch.stack([torch.randint(0, 134, (n, h, w), generator=g), torch.randint(0, 21, (n, h, w), generator=g),
                        torch.randint(0, 6, (n, h, w), generator=g), torch.randint(0, 3, (n, h, w), generator=g)], 1).to(torch.uint8)


def _step(m, x, pw, idx_ref):
    from mas_b200 import ops
    cb = m.quantize

    def fwd(z):                        # the quantiser's decision pinned, as in tests/test_host_logic_vq_cpu.py
        zq, loss = ops.VQGivenFn.apply(z, cb.embedding.weight, cb.beta, idx_ref)
        return zq, loss, idx_ref
    cb.forward = fwd
    m.zero_grad(set_to_none=True)
    dec, diff = m(x)
    loss = ops.BCELogitsFn.apply(dec, x, pw) + diff
    loss.backward()
    return dec.detach().clone(), loss.detach().clone(), {k: p.grad.clone() for k, p in m.named_parameters()}


def test_compact_vqseg_step_host_logic_against_oracle_and_dense_step(scene_emu):
    """The compact VQ-SEG step issues the scene entries (expansion for conv_in's forward and again for its weight gradient,
    the label-reading BCE pair) and never the dense map's pad copy or mas_bce_cl_*, with conv_in on the padded tensor route.
    It reproduces the dense step bit for bit and the CPU oracle."""
    from oracle import vqgan_oracle as O
    m, _, pw = _vqseg_model()
    lab = _labels()
    seg = torch.from_numpy(expand_np(lab.numpy()).transpose(0, 3, 1, 2).copy())
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    params = {k: v.requires_grad_(True) for k, v in sd.items() if v.is_floating_point() and "running" not in k}
    sd.update(params)
    dec_o, diff_o, idx_o = O.vqbase_forward(sd, VQSEG_DD, seg)
    lo = O.bce_loss_with_quant(diff_o, seg, dec_o)
    lo.backward()
    idx_ref = idx_o.view(-1)
    state = {k: v.clone() for k, v in m.state_dict().items()}
    first = len(scene_emu.names)
    dec_d, loss_d, g_d = _step(m, seg, pw, idx_ref)
    dense_names = scene_emu.names[first:]
    bn_d = {k: v.clone() for k, v in m.state_dict().items() if "running" in k}
    m.load_state_dict(state)
    first = len(scene_emu.names)
    dec_c, loss_c, g_c = _step(m, lab, pw, idx_ref)
    n = scene_emu.names[first:]
    assert n.count("mas_scene_expand") == 2 and n.count("mas_bce_scene_forward") == 1 and n.count("mas_bce_scene_backward") == 1
    assert not any(k in n for k in ("mas_nchw_to_nhwc_pad", "mas_bce_cl_forward", "mas_bce_cl_backward", "mas_bce_logits"))
    assert [k for k in n if not k.startswith(("mas_scene", "mas_bce"))] == [k for k in dense_names if not k.startswith(("mas_nchw", "mas_bce"))]
    assert torch.equal(dec_c, dec_d) and torch.equal(loss_c, loss_d)
    for k in g_d:
        assert torch.equal(g_c[k], g_d[k]), k
    for k, v in m.state_dict().items():
        if "running" in k:
            assert torch.equal(v, bn_d[k]), k
    assert rel_err(dec_c, dec_o) < 2e-3
    lo = float(lo.detach())
    assert abs(float(loss_c) - lo) < 2e-3 * abs(lo)
    for k, pr in params.items():
        assert rel_err(g_c[k], pr.grad) < 1e-2, k


def test_compact_conv_in_general_route_host_logic(scene_emu):
    """conv_in at a height off the tensor kernels' 16-row tile takes the general route: the compact map is expanded to the
    dense NCHW map for the forward and again for the weight gradient, and output and gradients equal the dense input's."""
    from mas_b200 import _lib as L, ops
    lab = _labels(2, 24, 16, seed=3)
    seg = torch.from_numpy(expand_np(lab.numpy()).transpose(0, 3, 1, 2).copy())
    g = torch.Generator().manual_seed(4)
    w0, b0 = torch.randn(128, 159, 3, 3, generator=g) / 40, torch.randn(128, generator=g)
    out = []
    for x in (seg, lab):
        first = len(scene_emu.names)
        wt, b = w0.clone().requires_grad_(True), b0.clone().requires_grad_(True)
        y = ops.Conv3x3Fn.apply(x, wt, b, None, L.CONV_S1, False)
        (y * torch.linspace(-1, 1, y.numel()).view(y.shape)).sum().backward()
        out.append((y.detach(), wt.grad, b.grad, scene_emu.names[first:]))
    (yd, gwd, gbd, nd), (yc, gwc, gbc, nc) = out
    assert "mas_nchw_to_nhwc_pad" not in nd and [k for k in nc if k != "mas_scene_expand"] == nd
    assert nc[0] == "mas_scene_expand" and nc[nc.index("mas_conv3x3_wgrad") - 1] == "mas_scene_expand" and nc.count("mas_scene_expand") == 2
    assert torch.equal(yc, yd) and torch.equal(gwc, gwd) and torch.equal(gbc, gbd)


def test_compact_bce_fallback_and_bad_inputs_host_logic(scene_emu):
    """Logits that are not the padded channels-last view take the generic kernel on the target expanded on the device; a
    compact target of the wrong extents, of non-159-channel logits, or a uint8 input to any other convolution raises."""
    from mas_b200 import _lib as L, ops
    lab = _labels(2, 8, 32)
    logits = torch.randn(2, 159, 8, 32)
    pw = torch.ones(159)
    seen = {}

    def bce_logits(lg, ls, tg, ts, pw_, loss, grad, gs, scale, ws, nb):
        seen["target"] = torch.from_numpy(_view4(tg, ts).copy())
        _f32(loss, 1)[0] = 0
    scene_emu.mas_bce_logits = bce_logits
    ops.BCELogitsFn.apply(logits, lab, pw)
    assert scene_emu.names[-2:] == ["mas_scene_expand", "mas_bce_logits"]
    assert torch.equal(seen["target"], torch.from_numpy(expand_np(lab.numpy())))
    with pytest.raises(RuntimeError):
        ops.BCELogitsFn.apply(logits, lab[:, :, :4], pw)
    with pytest.raises(RuntimeError):
        ops.BCELogitsFn.apply(logits[:, :158], lab, pw[:158])
    with pytest.raises(RuntimeError):
        ops.Conv3x3Fn.apply(lab, torch.randn(128, 158, 3, 3), None, None, L.CONV_S1, False)
    with pytest.raises(RuntimeError):
        ops.Conv3x3Fn.apply(lab, torch.randn(128, 159, 3, 3), None, None, L.CONV_S2, False)
