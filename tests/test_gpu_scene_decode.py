"""The output side of compact scene maps on the H100: mas_scene_decode against the numpy statement of the rule
(tests/test_scene_decode_cpu.py) bit for bit on every layout, the pack -> expand -> decode round trip, mas_scene_confusion
against numpy.bincount, and VQBASE.decode_scene on seeded VQ-SEG models."""
import numpy as np
import pytest
import torch

from test_scene_decode_cpu import _hard_logits, confusion_np, decode_np

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _logits(b, h, w, seed):
    """Random logits around the decision boundary, the hard cases of the CPU test (ties, zeros, NaNs, infinities) in the
    first rows of image 0."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, 159, h, w, generator=g) * 2 - 1.5
    hard = torch.from_numpy(_hard_logits(seed, b=2, h=2, w=7))[:1, :, :h, :w]
    x[:1, :, :hard.shape[2], :hard.shape[3]] = hard
    return x


def _layout(x, layout):
    """x on the device in the given layout (same logical values)."""
    b, c, h, w = x.shape
    if layout == "padded_cl":                           # the decoder's output: channels-last, pitch 160, pad channel NaN
        base = torch.full((b, h, w, 160), float("nan"), device=DEV)
        base[..., :159] = x.permute(0, 2, 3, 1).to(DEV)
        return base.permute(0, 3, 1, 2)[:, :159]
    if layout == "nchw":
        return x.to(DEV)
    if layout == "strided":                             # every other column of a wider NCHW tensor, channels 3..161 of 170
        big = torch.randn(b, 170, h, 2 * w, device=DEV)
        big[:, 3:162, :, ::2] = x.to(DEV)
        return big[:, 3:162, :, ::2]
    raise ValueError(layout)


CASES = [("padded_cl", 2, 16, 64), ("padded_cl", 2, 9, 45), ("padded_cl", 1, 8, 32), ("padded_cl", 33, 4, 40),
         ("nchw", 2, 16, 64), ("nchw", 1, 5, 45), ("nchw", 33, 3, 20), ("strided", 2, 6, 37)]


@pytest.mark.parametrize("layout,b,h,w", CASES)
def test_decode_matches_the_rule_bit_for_bit(layout, b, h, w):
    from mas_b200 import scene
    x = _logits(b, h, w, seed=b * 1000 + h * 10 + w)
    lg = _layout(x, layout)
    got = scene.decode(lg)
    assert got.dtype == torch.uint8 and got.shape == (b, 4, h, w) and got.is_contiguous() and got.device == lg.device
    want = decode_np(x.numpy())
    assert np.array_equal(got.cpu().numpy(), want)
    assert torch.equal(scene.decode(lg), got)              # the same bytes on every call
    if layout == "padded_cl":
        assert (want[:, 0] > 0).any() and (want[:, 0] == 0).any() and (want[:, 3] == 1).any()


def test_pack_expand_decode_round_trip():
    """pack -> mas_scene_expand (dense NCHW and the padded channels-last operand) -> decode returns the packed planes, edge
    counts of 2 as 1."""
    from mas_b200 import ops, scene
    rng = np.random.default_rng(3)
    shape = (3, 24, 40)
    a = (rng.integers(-1, 133, shape), rng.integers(-1, 20, shape), rng.integers(0, 6, shape), rng.integers(0, 3, shape))
    a[0][0, 0, :2], a[1][0, 0, :2], a[2][0, 0, :2], a[3][0, 0, :3] = (-1, 132), (-1, 19), (0, 5), (0, 1, 2)
    lab = scene.pack(*a)
    want = lab.clone()
    want[:, 3].clamp_(max=1)
    labd = lab.to(DEV)
    dense, padded = ops.scene_expand(labd), ops.scene_expand(labd, 160)[:, :159]   # NCHW, and the decoder's padded view
    for d in (dense, padded):
        assert torch.equal(scene.decode(d).cpu(), want)
    got = scene.unpack(scene.decode(padded).cpu())
    assert all(np.array_equal(g, w) for g, w in zip(got[:3], a[:3])) and np.array_equal(got[3], np.minimum(a[3], 1))


@pytest.mark.parametrize("b,h,w", [(3, 17, 45), (2, 64, 64), (4, 256, 256)])
def test_confusion_matches_bincount(b, h, w):
    """Random maps with out-of-range bytes in both maps, and maps that are mostly "none" (the ballot-counted cell)."""
    from mas_b200 import scene
    g = torch.Generator().manual_seed(b * h)
    hi = torch.tensor([134, 21, 6, 3]).view(1, 4, 1, 1)
    target = (torch.rand(b, 4, h, w, generator=g) * hi).to(torch.uint8)
    pred = (torch.rand(b, 4, h, w, generator=g) * hi).to(torch.uint8)
    target[torch.rand(b, 4, h, w, generator=g) < 0.6] = 0
    pred[torch.rand(b, 4, h, w, generator=g) < 0.6] = 0
    bad_t = torch.rand(b, 4, h, w, generator=g) < 0.01
    bad_p = torch.rand(b, 4, h, w, generator=g) < 0.01
    target[bad_t] = (torch.randint(0, 256, (int(bad_t.sum()),), generator=g)).to(torch.uint8) | 0x80
    pred[bad_p] = 255
    want = confusion_np(pred.view(b, 4, -1).numpy(), target.view(b, 4, -1).numpy())
    conf = scene.confusion(pred.to(DEV), target.to(DEV))
    got = np.concatenate([conf[k].cpu().numpy().ravel() for k in scene.GROUPS] + [conf["out_of_range"].cpu().numpy().ravel()])
    assert np.array_equal(got, want)
    assert int(conf["out_of_range"]) > 0 and int(conf["panoptic"].sum()) + int(conf["out_of_range"]) >= b * h * w
    again = scene.confusion(pred.to(DEV), target.to(DEV))
    assert all(torch.equal(again[k], conf[k]) for k in conf)
    same = scene.confusion(target.to(DEV), target.to(DEV))       # a map against itself: diagonal matrices
    for k in scene.GROUPS:
        m = same[k].cpu()
        assert torch.equal(m, torch.diag(torch.diag(m)))


TINY_SEG = dict(z_channels=32, in_channels=159, out_channels=159, channels=[32, 32, 64], num_res_blocks=1, resolution=16,
                attn_resolutions=[8], dropout=0.0)
TC_SEG = dict(z_channels=64, in_channels=159, out_channels=159, channels=[128, 128], num_res_blocks=1, resolution=64,
              attn_resolutions=[], dropout=0.0)


@pytest.mark.parametrize("name,dd,grid,f", [("tiny", TINY_SEG, 8, 2), ("tc", TC_SEG, 32, 1)])
def test_decode_scene_is_decode_of_decode_code(name, dd, grid, f):
    from mas_b200 import _lib, scene
    from models import VQBASE
    torch.manual_seed(0)
    m = VQBASE(dd, 128, dd["z_channels"], 10, 100)
    with torch.no_grad():
        m.quantize.embedding.weight.normal_()
    m = m.to(DEV).train()
    tok = torch.randint(0, 128, (3, grid, grid), generator=torch.Generator().manual_seed(1)).to(DEV)
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    modes = {n: mod.training for n, mod in m.named_modules()}
    q, res = m.quantize.q_counter, m.quantize.reservoir
    with torch.enable_grad(), _lib.launch_trace() as trace:
        got = m.decode_scene(tok)
        torch.cuda.synchronize()
    assert "scene_decode_cl" in trace, trace[-5:]
    assert got.dtype == torch.uint8 and got.shape == (3, 4, grid * f, grid * f)
    assert not got.requires_grad and got.grad_fn is None
    with torch.no_grad():
        dec = m.decode_code(tok)
    assert dec.stride(1) == 1                                  # the decoder's channels-last view
    assert torch.equal(got, scene.decode(dec))
    assert np.array_equal(got.cpu().numpy(), decode_np(dec.cpu().numpy()))
    now = m.state_dict()
    for k, v in sd.items():
        assert torch.equal(now[k], v), k
    assert {n: mod.training for n, mod in m.named_modules()} == modes
    assert m.quantize.q_counter == q and m.quantize.reservoir is res and all(p.grad is None for p in m.parameters())
    # the evaluation chain: encode_code -> decode_scene -> confusion -> iou
    lab = scene.decode(m.decode_code(tok))
    m.eval()
    rec = m.decode_scene(m.encode_code(lab))
    r = scene.iou(scene.confusion(rec, lab))
    assert set(r) == set(scene.GROUPS) and r["panoptic"]["iou"].shape == (134,)
    c = scene.confusion(rec, lab)
    assert int(c["out_of_range"]) == 0 and int(c["panoptic"].sum()) == lab.shape[0] * lab.shape[2] * lab.shape[3]


def test_validation_on_the_device():
    from mas_b200 import scene
    from models import VQBASE
    x = torch.zeros(1, 159, 8, 8, device=DEV)
    lab = torch.zeros(1, 4, 8, 8, dtype=torch.uint8, device=DEV)
    for f in (lambda: scene.decode(x.cpu()), lambda: scene.decode(x.half()), lambda: scene.decode(x[:, :100]),
              lambda: scene.confusion(lab, lab.cpu()), lambda: scene.confusion(lab, lab[..., :4])):
        with pytest.raises(ValueError):
            f()
    torch.manual_seed(0)
    img = VQBASE(dict(TINY_SEG, in_channels=3, out_channels=3), 64, 32, 10, 100).to(DEV)
    with pytest.raises(ValueError):
        img.decode_scene(torch.zeros(1, 8, 8, dtype=torch.int64, device=DEV))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs a second GPU")
def test_confusion_on_each_device_of_one_process():
    """The shared-memory opt-in of the confusion kernel is made per device: the same maps on cuda:0, then cuda:1 (not the
    current device), give the same counts."""
    from mas_b200 import scene
    g = torch.Generator().manual_seed(5)
    hi = torch.tensor([134, 21, 6, 3]).view(1, 4, 1, 1)
    pred, target = ((torch.rand(2, 4, 32, 48, generator=g) * hi).to(torch.uint8) for _ in range(2))
    want = confusion_np(pred.view(2, 4, -1).numpy(), target.view(2, 4, -1).numpy())
    for d in (torch.device("cuda:0"), torch.device("cuda:1")):
        conf = scene.confusion(pred.to(d), target.to(d))
        got = np.concatenate([conf[k].cpu().numpy().ravel() for k in scene.GROUPS] + [conf["out_of_range"].cpu().numpy().ravel()])
        assert conf["panoptic"].device == d and np.array_equal(got, want)
