"""The output side of compact scene maps without a GPU: the decoding rule of mas_scene_decode restated in numpy and checked
against a direct torch statement of it and against an emulation of the kernel's order-key warp reduction; unpack as the exact
inverse of pack; scene.iou on hand-written matrices; and the host logic of scene.decode / scene.confusion /
VQBASE.decode_scene above the emulated C-ABI of tests/test_host_logic_vq_cpu.py (the calls and strides they issue, no aten
arithmetic, every ValueError before any call).  The kernels are tested on the GPU (tests/test_gpu_scene_decode.py)."""
import ctypes

import numpy as np
import pytest
import torch

from test_host_logic_vq_cpu import VQSEG_DD, _addr, _view4, vq_emu  # noqa: F401  (vq_emu: fixture)
from test_scene_maps_cpu import SceneEmu, expand_np, _u8
from test_seg_mse_loss_cpu import PLUMBING, TorchOps

GROUPS = ((0, 133), (133, 153), (153, 158))


def decode_np(x):
    """The rule (include/mas_b200.h, mas_scene_decode) on [B, 159, H, W] float32 -> [B, 4, H, W] uint8: per one-hot group
    1 + argmax (first maximum; NaN never wins) when the maximum is > 0, else 0; edges x[158] > 0."""
    x = np.asarray(x, dtype=np.float32)
    out = np.zeros((x.shape[0], 4) + x.shape[2:], dtype=np.uint8)
    for p, (a, b) in enumerate(GROUPS):
        g = np.where(np.isnan(x[:, a:b]), -np.inf, x[:, a:b])
        out[:, p] = np.where(g.max(1) > 0, g.argmax(1) + 1, 0)
    out[:, 3] = x[:, 158] > 0
    return out


def decode_torch(x):
    """The same rule as a user would write it in torch: slice, argmax, threshold and stack."""
    planes = []
    for a, b in GROUPS:
        g = x[:, a:b].nan_to_num(nan=float("-inf"), posinf=float("inf"), neginf=float("-inf"))
        planes.append(torch.where(g.amax(1) > 0, g.argmax(1) + 1, 0))
    planes.append((x[:, 158] > 0).long())
    return torch.stack(planes, 1).to(torch.uint8)


def _keys(x):
    """The kernel's order keys: float bits mapped monotonically onto uint32, -0 onto +0, NaN to 0."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    k = np.where(u & 0x80000000, ~u & 0xFFFFFFFF, u | 0x80000000)
    k = np.where(x == 0, 0x80000000, k)
    return np.where(np.isnan(x), 0, k)


def decode_warp_emu(x):
    """scene.cu's channels-last kernel, lane by lane: lane l holds channels l + 32k; per lane the first best key, then the warp
    max of the keys and the min channel holding it (redux.sync max / min)."""
    x = np.asarray(x, dtype=np.float32)
    B, _, H, W = x.shape
    k = _keys(np.concatenate([x, np.zeros((B, 1, H, W), np.float32)], 1))    # + the pad channel, never used
    out = np.zeros((B, 4, H, W), dtype=np.uint8)
    ch = np.arange(160).reshape(5, 32)                                        # [k, lane]
    kk = k.transpose(0, 2, 3, 1).reshape(B, H, W, 5, 32)
    pan = np.where(ch < 133, kk, 0)
    best = np.zeros((B, H, W, 32), np.uint64)
    bi = np.tile(np.arange(32), (B, H, W, 1))
    for j in range(5):
        upd = pan[..., j, :] > best if j else np.ones_like(best, dtype=bool)
        best = np.where(upd, pan[..., j, :], best)
        bi = np.where(upd, ch[j], bi)
    lane = np.arange(32)
    for p, (keys, idx) in enumerate(((best, bi), (np.where((lane >= 5) & (lane < 25), kk[..., 4, :], 0), lane - 5),
                                     (np.where((lane >= 25) & (lane < 30), kk[..., 4, :], 0), lane - 25))):
        m = keys.max(-1, keepdims=True)
        i = np.where(keys == m, idx, 1 << 32).min(-1)
        out[:, p] = np.where(m[..., 0] > 0x80000000, i + 1, 0)
    out[:, 3] = kk[..., 4, 30] > 0x80000000
    return out


def _hard_logits(seed=0, b=2, h=6, w=7):
    """Random logits with exact ties at the group maximum, maxima of exactly +0 / -0, NaNs, all-NaN groups, infinities."""
    rng = np.random.default_rng(seed)
    x = rng.normal(size=(b, 159, h, w)).astype(np.float32)
    x[0, :, 0, 0] = -1.0
    x[0, [5, 17, 140, 150, 155, 157], 0, 0] = 2.5                   # ties in every group
    x[0, :, 0, 1] = -3.0
    x[0, [7, 140, 154, 158], 0, 1] = 0.0                            # maximum exactly 0: none, no edge
    x[0, [3, 135, 156], 0, 2] = -0.0
    x[0, :, 0, 2] = np.where(x[0, :, 0, 2] > 0, -x[0, :, 0, 2], x[0, :, 0, 2])
    x[0, :, 0, 3] = np.nan                                          # all-NaN pixel
    x[0, 0:133, 0, 4] = -1.0
    x[0, 0:133:2, 0, 4] = np.nan                                    # NaN beside a positive maximum
    x[0, 11, 0, 4] = 0.7
    x[0, 133:153, 0, 5] = np.nan                                    # one all-NaN group, the others real
    x[0, 153:158, 0, 5] = np.nan
    x[0, 158, 0, 5] = np.nan
    x[0, [20, 21], 0, 6] = np.inf                                   # tied infinities
    x[0, 0:133, 1, 0] = -np.inf
    x[1, :, 1] = 0.0                                                # a row of +0 / -0 only
    x[1, ::3, 1] = -0.0
    return x


def _dense(rng, b, h, w):
    lab = np.stack([rng.integers(0, 134, (b, h, w)), rng.integers(0, 21, (b, h, w)), rng.integers(0, 6, (b, h, w)),
                    rng.integers(0, 3, (b, h, w))], 1).astype(np.uint8)
    return lab, expand_np(lab).transpose(0, 3, 1, 2).copy()


def test_rule_numpy_torch_and_warp_emulation_agree():
    for seed in range(3):
        x = _hard_logits(seed)
        want = decode_np(x)
        assert np.array_equal(decode_torch(torch.from_numpy(x)).numpy(), want)
        assert np.array_equal(decode_warp_emu(x), want)
    x = _hard_logits(0)
    got = decode_np(x)
    assert list(got[0, :, 0, 0]) == [6, 8, 3, 0]                     # ties -> the lowest channel of each group
    assert list(got[0, :, 0, 1]) == [0, 0, 0, 0] and list(got[0, :, 0, 2]) == [0, 0, 0, 0]
    assert list(got[0, :, 0, 3]) == [0, 0, 0, 0]                     # all NaN
    assert got[0, 0, 0, 4] == 12 and list(got[0, 1:, 0, 5]) == [0, 0, 0]
    assert got[0, 0, 0, 6] == 21 and got[0, 0, 1, 0] == 0 and not got[1, :, 1].any()


def test_dense_maps_decode_to_their_planes_edges_clipped():
    rng = np.random.default_rng(4)
    lab, dense = _dense(rng, 3, 5, 9)
    lab[0, :, 0, :3] = [[0, 133, 7], [0, 20, 3], [0, 5, 1], [0, 1, 2]]
    dense = expand_np(lab).transpose(0, 3, 1, 2).copy()
    want = lab.copy()
    want[:, 3] = np.minimum(want[:, 3], 1)
    for f in (decode_np, decode_warp_emu, lambda d: decode_torch(torch.from_numpy(d)).numpy()):
        assert np.array_equal(f(dense), want)


def test_unpack_inverts_pack():
    from mas_b200 import scene
    rng = np.random.default_rng(2)
    shape = (3, 6, 11)
    a = (rng.integers(-1, 133, shape), rng.integers(-1, 20, shape), rng.integers(0, 6, shape), rng.integers(0, 3, shape))
    a[0][0, 0, :2], a[1][0, 0, :2], a[2][0, 0, :2], a[3][0, 0, :2] = (-1, 132), (-1, 19), (0, 5), (0, 2)
    got = scene.unpack(scene.pack(*a))
    assert all(g.dtype == np.int64 and np.array_equal(g, w) for g, w in zip(got, a))
    one = scene.unpack(scene.pack(*(v[1] for v in a)).numpy())          # one image, a numpy array
    assert all(np.array_equal(g, w[1]) for g, w in zip(one, a))


@pytest.mark.parametrize("plane,value", [(0, 134), (0, 255), (1, 21), (2, 6), (3, 3), (3, 200)])
def test_unpack_rejects_bytes_out_of_range(plane, value):
    from mas_b200 import scene
    lab = torch.zeros(2, 4, 3, 5, dtype=torch.uint8)
    lab[1, plane, 2, 4] = value
    with pytest.raises(ValueError):
        scene.unpack(lab)


def test_unpack_rejects_bad_arrays():
    from mas_b200 import scene
    for bad in (np.zeros((4, 3, 5), np.int64), np.zeros((3, 3, 5), np.uint8), np.zeros((2, 5), np.uint8),
                np.zeros((0, 4, 3, 5), np.uint8), np.zeros((1, 1, 4, 3, 5), np.uint8)):
        with pytest.raises(ValueError):
            scene.unpack(bad)


def test_iou_on_hand_written_matrices():
    from mas_b200 import scene
    pan = np.zeros((134, 134), np.int64)
    pan[0, 0], pan[1, 1], pan[1, 2], pan[2, 1], pan[3, 3] = 50, 6, 2, 1, 4    # class 1: 6 / (6 + 1 + 2); class 3: 1
    pan[5, 0] = 3                                                             # class 5: missed entirely -> 0
    hum = np.zeros((21, 21), np.int64)                                        # empty: every union empty
    face = np.zeros((6, 6), np.int64)
    face[0, 0] = 9
    face[0, 4] = 1                                                            # a false positive only -> IoU 0
    edges = np.array([[10, 2], [3, 5]], np.int64)
    r = scene.iou({"panoptic": torch.from_numpy(pan), "human": hum, "face": face, "edges": edges})
    p = r["panoptic"]["iou"]
    assert p[1] == pytest.approx(6 / 9) and p[2] == 0.0 and p[3] == 1.0 and p[5] == 0.0 and p[0] == pytest.approx(50 / 53)
    assert np.isnan(p[4]) and np.isnan(p[133])
    assert r["panoptic"]["miou"] == pytest.approx((6 / 9 + 0 + 1 + 0) / 4)
    assert np.isnan(r["human"]["iou"]).all() and np.isnan(r["human"]["miou"])
    assert r["face"]["iou"][4] == 0.0 and r["face"]["miou"] == 0.0 and r["face"]["iou"][0] == 0.9
    assert r["edges"]["miou"] == pytest.approx(5 / 10) and r["edges"]["iou"][0] == pytest.approx(10 / 15)
    with pytest.raises(ValueError):
        scene.iou({"panoptic": pan[:5], "human": hum, "face": face, "edges": edges})


# ------------------------------------------------------------------------------------------------ host logic over the C-ABI
def confusion_np(pred, target):
    """Documented semantics of mas_scene_confusion on [B, 4, P] uint8 maps -> the 18438 counts."""
    out = []
    bad = np.zeros(target[:, 0].size, dtype=bool)
    for p, k in enumerate((134, 21, 6, 2)):
        t, y = target[:, p].astype(np.int64).ravel(), pred[:, p].astype(np.int64).ravel()
        hi = 2 if p == 3 else k - 1
        ok = (t <= hi) & (y <= hi)
        bad |= ~ok
        if p == 3:
            t, y = np.minimum(t, 1), np.minimum(y, 1)
        out.append(np.bincount(t[ok] * k + y[ok], minlength=k * k))
    return np.concatenate(out + [np.array([bad.sum()])]).astype(np.int64)


class DecodeEmu(SceneEmu):
    def mas_scene_decode(self, x, xs, planes):
        assert xs.c == 159
        v = _view4(x, xs).transpose(0, 3, 1, 2)
        _u8(planes, xs.n * 4 * xs.h * xs.w)[:] = decode_np(v).ravel()
        self.decode_t4 = (xs.n, xs.h, xs.w, xs.c, xs.sn, xs.sh, xs.sw, xs.sc)

    def mas_scene_confusion(self, pred, target, P, B, conf, ws, ws_bytes):
        n = B * 4 * P
        c = confusion_np(_u8(pred, n).reshape(B, 4, P), _u8(target, n).reshape(B, 4, P))
        np.ctypeslib.as_array((ctypes.c_int64 * 18438).from_address(_addr(conf)))[:] = c


@pytest.fixture
def decode_emu(vq_emu, monkeypatch):  # noqa: F811
    from mas_b200 import ops, scene
    from models import vqvae
    e = DecodeEmu()
    monkeypatch.setattr(ops.L, "call", e)
    monkeypatch.setattr(ops, "_need_cuda", lambda x, dtype=None: None)
    monkeypatch.setattr(scene, "_kernel_device", lambda t: True)
    monkeypatch.setattr(vqvae, "_kernel_device", lambda t: True)
    return e


def test_decode_and_confusion_host_logic(decode_emu):
    """scene.decode passes the logits' own strides (padded channels-last view, NCHW, a strided slice) and returns what the rule
    gives; scene.confusion passes the contiguous maps and splits the counts; neither runs aten arithmetic."""
    from mas_b200 import scene
    x = torch.from_numpy(_hard_logits(1, b=2, h=4, w=7))
    base = torch.zeros(2, 4, 7, 160)
    base[..., :159] = x.permute(0, 2, 3, 1)
    base[..., 159] = float("nan")                                   # the pad channel may hold anything
    wide = torch.from_numpy(_hard_logits(2, b=2, h=4, w=14))
    for lg, t4 in ((base.permute(0, 3, 1, 2)[:, :159], (2, 4, 7, 159, 4 * 7 * 160, 7 * 160, 160, 1)),
                   (x, (2, 4, 7, 159, 159 * 28, 7, 1, 28)),
                   (wide[..., ::2], (2, 4, 7, 159, 159 * 56, 14, 2, 56))):
        first = len(decode_emu.names)
        with TorchOps() as rec:
            got = scene.decode(lg)
        assert decode_emu.names[first:] == ["mas_scene_decode"] and decode_emu.decode_t4 == t4
        assert rec.ops <= PLUMBING, rec.ops - PLUMBING
        assert got.dtype == torch.uint8 and got.shape == (2, 4, 4, 7) and got.is_contiguous()
        assert np.array_equal(got.numpy(), decode_np(lg.numpy()))
    rng = np.random.default_rng(7)
    target, _ = _dense(rng, 2, 5, 8)
    target[0, 3, 0, 0] = 9                                           # out of range: counted apart
    target[1, 2, 2, 3] = 77
    pred = decode_np(_dense(rng, 2, 5, 8)[1])
    pred[0, 1, 0, 0] = 200                                           # the same pixel as the first: counted once
    first = len(decode_emu.names)
    with TorchOps() as rec:
        conf = scene.confusion(torch.from_numpy(pred), torch.from_numpy(target).transpose(2, 3).contiguous().transpose(2, 3))
    assert decode_emu.names[first:] == ["mas_scene_confusion"]
    assert rec.ops <= PLUMBING, rec.ops - PLUMBING
    want = confusion_np(pred.reshape(2, 4, -1), target.reshape(2, 4, -1))
    got = np.concatenate([conf[g].numpy().ravel() for g in scene.GROUPS] + [conf["out_of_range"].numpy().ravel()])
    assert np.array_equal(got, want) and int(conf["out_of_range"]) == 2
    assert conf["panoptic"].shape == (134, 134) and conf["edges"].shape == (2, 2) and int(conf["panoptic"].sum()) == 80
    assert [int(conf[g].sum()) for g in ("human", "face", "edges")] == [79, 79, 79]   # the other planes are still counted


def _seg_model(dd):
    from models import VQBASE
    torch.manual_seed(0)
    m = VQBASE(dd, 128, 64, 10, 100)
    with torch.no_grad():
        m.quantize.embedding.weight.normal_()
    return m.train()


def test_decode_scene_host_logic_and_no_side_effects(decode_emu):
    """decode_scene = decode_code's calls, then one mas_scene_decode on the decoder's output as it is (its strides); in train
    mode nothing of the module changes and no graph is recorded."""
    from mas_b200 import scene
    m = _seg_model(dict(VQSEG_DD, channels=[32, 32], resolution=16))
    tok = torch.randint(0, 128, (2, 16, 16), generator=torch.Generator().manual_seed(1))
    m.decode_code(tok)                                              # packs and caches the weight images
    first = len(decode_emu.names)
    dec = m.decode_code(tok)
    ref_names = decode_emu.names[first:]
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    modes = {n: mod.training for n, mod in m.named_modules()}
    q, res = m.quantize.q_counter, m.quantize.reservoir
    first = len(decode_emu.names)
    with torch.enable_grad():
        got = m.decode_scene(tok)
    assert decode_emu.names[first:] == ref_names + ["mas_scene_decode"]
    assert decode_emu.decode_t4 == tuple(getattr(scene.L.t4(dec), f) for f in ("n", "h", "w", "c", "sn", "sh", "sw", "sc"))
    assert got.dtype == torch.uint8 and got.shape == (2, 4, 16, 16) and not got.requires_grad and got.grad_fn is None
    assert np.array_equal(got.numpy(), decode_np(dec.detach().numpy()))
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k
    assert {n: mod.training for n, mod in m.named_modules()} == modes
    assert m.quantize.q_counter == q and m.quantize.reservoir is res and all(p.grad is None for p in m.parameters())


def test_every_value_error_fires_before_any_call(decode_emu, monkeypatch):
    from mas_b200 import scene
    from models import vqvae
    x = torch.zeros(1, 159, 4, 4)
    lab = torch.zeros(1, 4, 4, 4, dtype=torch.uint8)
    seg = _seg_model(dict(VQSEG_DD, channels=[32, 32], resolution=16))
    img = _seg_model(dict(VQSEG_DD, channels=[32, 32], resolution=16, in_channels=3, out_channels=3))
    tok = torch.zeros(1, 2, 2, dtype=torch.int64)
    cases = [lambda: scene.decode(x.double()), lambda: scene.decode(x.half()), lambda: scene.decode(x[:, :158]),
             lambda: scene.decode(torch.zeros(1, 160, 4, 4)), lambda: scene.decode(x[0]), lambda: scene.decode(x.numpy()),
             lambda: scene.decode(x[:0]), lambda: scene.decode(x[:, :, :0]), lambda: scene.decode(x[..., :0]),
             lambda: scene.decode(torch.zeros(1, 159, 65536, 1)),
             lambda: scene.confusion(lab, lab.float()), lambda: scene.confusion(lab.long(), lab),
             lambda: scene.confusion(lab, lab[:, :3]), lambda: scene.confusion(lab[:0], lab[:0]),
             lambda: scene.confusion(lab[..., :0], lab[..., :0]), lambda: scene.confusion(lab, lab[..., :3]),
             lambda: scene.confusion(lab[0], lab[0]),
             lambda: img.decode_scene(tok), lambda: seg.decode_scene(tok.int()), lambda: seg.decode_scene(tok[0]),
             lambda: seg.decode_scene(tok[:0]), lambda: seg.decode_scene(tok.float())]
    first = len(decode_emu.names)
    for f in cases:
        with pytest.raises(ValueError):
            f()
    monkeypatch.setattr(scene, "_kernel_device", lambda t: t.is_cuda)
    monkeypatch.setattr(vqvae, "_kernel_device", lambda t: t.is_cuda)
    for f in (lambda: scene.decode(x), lambda: scene.confusion(lab, lab), lambda: seg.decode_scene(tok)):
        with pytest.raises(ValueError):                              # CPU tensors
            f()
    assert decode_emu.names[first:] == []
