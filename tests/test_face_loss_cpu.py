"""VGGFace2 face-loss drop-in (losses/face_loss.py) without a GPU: parameter layout and seeded initialisation against the
real reference (tests/golden/face_loss.pt), resolution of the `losses` package next to a reference checkout, the refusals,
the faces[:6] pairing rule and the crop table, and the fp64 restatement of tests/face_common.py against every golden case.
The kernels are tested on the GPU (tests/test_gpu_face_loss.py)."""
import hashlib
import subprocess
import sys
import textwrap

import pytest
import torch

from conftest import PKG, rel_err
from face_common import build_face_loss, case_inputs, load_golden, restated_loss, seeded_face_loss


@pytest.fixture(scope="module")
def golden():
    return load_golden()


def _sha(t):
    return hashlib.sha256(t.detach().contiguous().numpy().tobytes()).hexdigest()


@pytest.mark.parametrize("name", ["a", "b", "c"])
def test_state_dict_and_seeded_init_match_reference(golden, name):
    case = golden[name]
    m, checks = seeded_face_loss(case)
    sd = m.state_dict()
    assert list(sd) == list(case["init"]) and len(sd) == 318
    for k, v in sd.items():
        ref = case["init"][k]
        assert tuple(v.shape) == ref["shape"] and str(v.dtype) == ref["dtype"], k
        assert _sha(v) == ref["sha256"], k
    assert checks == case["fill_checks"]
    assert sum(p.numel() for p in m.parameters()) == 23_508_032
    img, rec = case_inputs(case)
    assert _sha(torch.cat([img, rec])) == case["images_sha256"]


def test_checkpoints_load_both_ways(tmp_path):
    import losses.face_loss as fl
    m = build_face_loss()
    assert not m.training and not any(p.requires_grad for p in m.parameters())
    with torch.no_grad():
        for p in m.parameters():
            p.normal_()
    path = tmp_path / "w.pt"
    torch.save(m.state_dict(), path)
    saved = fl.WEIGHTS
    fl.WEIGHTS = str(path)
    try:
        m2 = fl.FaceLoss()
    finally:
        fl.WEIGHTS = saved
    for (k, a), (k2, b) in zip(m.state_dict().items(), m2.state_dict().items()):
        assert k == k2 and torch.equal(a, b), k


def test_missing_weight_file_names_the_variable(tmp_path):
    import losses.face_loss as fl
    with pytest.raises(FileNotFoundError, match="MAS_FACE_LOSS_WEIGHTS"):
        fl.load_weights(str(tmp_path / "absent.pt"))


def test_losses_package_resolves_next_to_reference(tmp_path):
    ref = tmp_path / "ref" / "losses"
    ref.mkdir(parents=True)
    (ref / "__init__.py").write_text("from .loss_img import VQLPIPSWithDiscriminator\n")
    (ref / "loss_img.py").write_text("from .face_loss import FaceLoss\nclass VQLPIPSWithDiscriminator:\n    pass\n")
    (ref / "face_loss.py").write_text("raise ImportError('the reference face loss must not be picked up')\n")
    prog = textwrap.dedent("""
        import sys
        sys.path[:0] = [%r, %r]
        import losses.face_loss as f
        assert "torchvision" not in sys.modules and "losses.lpips" not in sys.modules
        assert "losses.discriminator" not in sys.modules
        import losses.loss_img as li
        assert li.FaceLoss is f.FaceLoss and f.__file__.startswith(%r)
        import losses.lpips, losses.discriminator
        assert "torchvision" not in sys.modules
        print("ok")
    """) % (PKG, str(tmp_path / "ref"), PKG)
    r = subprocess.run([sys.executable, "-c", prog], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stderr
    prog = "import sys; sys.path[:0] = [%r]; import losses.lpips, losses.discriminator; " \
           "assert 'losses.face_loss' not in sys.modules; print('ok')" % PKG
    r = subprocess.run([sys.executable, "-c", prog], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.strip() == "ok", r.stderr


def test_refusals():
    m = build_face_loss()
    img = torch.zeros(1, 3, 64, 64)
    box = [[[0, 0, 32, 32]]]
    m.train()
    with pytest.raises(RuntimeError, match="training mode"):
        m(img, img, box)
    m.eval()
    m.layer2[0].conv2.weight.requires_grad_(True)
    with pytest.raises(RuntimeError, match="requires_grad=False"):
        m(img, img, box)
    m.layer2[0].conv2.weight.requires_grad_(False)
    for bad in ([[[10, 0, 10, 32]]], [[[0, 20, 32, 5]]]):
        with pytest.raises(ValueError, match="extent"):
            m(img, img, bad)
    # no kernels on the CPU: the forward itself refuses loudly
    with pytest.raises(RuntimeError):
        m(img, img, box)
    # no faces: the reference's img.new_tensor(0)
    z = m(img, img, [[]])
    assert z.dim() == 0 and float(z) == 0.0 and not z.requires_grad


def test_create_graph_is_refused():
    from mas_b200 import ops

    class Ctx:
        needs_input_grad = (False, True)
        J = None
    with torch.enable_grad(), pytest.raises(RuntimeError, match="create_graph"):
        ops.FaceLossFn.backward(Ctx(), torch.ones(()))


EXPECTED_PAIRS = {
    0: ([], []),
    1: ([("gt", 0)], [("gen", 0)]),
    2: ([("gt", 0), ("gt", 1)], [("gen", 0), ("gen", 1)]),
    3: ([("gt", 0), ("gt", 1), ("gt", 2)], [("gen", 0), ("gen", 1), ("gen", 2)]),
    4: ([("gt", 0), ("gt", 1), ("gt", 2)], [("gt", 3), ("gen", 0), ("gen", 1)]),
    5: ([("gt", 0), ("gt", 1), ("gt", 2)], [("gt", 3), ("gt", 4), ("gen", 0)]),
    6: ([("gt", 0), ("gt", 1), ("gt", 2)], [("gt", 3), ("gt", 4), ("gt", 5)]),
    7: ([("gt", 0), ("gt", 1), ("gt", 2)], [("gt", 3), ("gt", 4), ("gt", 5)]),
}


@pytest.mark.parametrize("n", range(8))
def test_pairing_rule(n):
    from mas_b200 import ops
    used = [("gt" if s == 0 else "gen", k) for s, k in ops.face_pairing(n)]
    half = len(used) // 2
    assert (used[:half], used[half:]) == EXPECTED_PAIRS[n]
    boxes = [[[i, i, i + 20, i + 30] for i in range(n)]]
    plan = ops.FacePlan((1, 3, 64, 64), (1, 3, 64, 64), boxes)
    assert plan.F == len(used) and [(f[0], f[2]) for f in plan.faces] == [(s, k) for s, k in ops.face_pairing(n)]
    # only the crops whose gradient is wanted are kept for the backward
    ngt = sum(1 for s, _ in ops.face_pairing(n) if s == 0)
    assert plan.span(False, True) == (ngt, plan.F) and plan.span(True, False) == (0, ngt)


def test_zip_truncates_like_the_reference():
    from mas_b200 import ops
    plan = ops.FacePlan((2, 3, 64, 64), (3, 3, 64, 64), [[[0, 0, 10, 10]], [[0, 0, 12, 12]], [[0, 0, 14, 14]]])
    assert plan.n == 2


def _crop_table_gather(plan, img, rec):
    """The crops the table describes, gathered in fp64 on the host exactly as mas_face_prepare reads them."""
    tab, wts = plan.tab.tolist(), plan.wts.double()
    out = torch.zeros(plan.F, 3, 254, 254, dtype=torch.float64)
    for f in range(plan.F):
        src, side, top, left, ch, cw, ky, kx, o_sy, o_sx, o_ay, o_ax, o_wy, o_wx = tab[14 * f:14 * f + 14]
        im = (rec if side else img)[src].double()
        H, W = im.shape[1:]
        Wy = torch.zeros(254, H, dtype=torch.float64)
        Wx = torch.zeros(254, W, dtype=torch.float64)
        for M, o_s, o_w, k, ext, org, lim in ((Wy, o_sy, o_wy, ky, ch, top, H), (Wx, o_sx, o_wx, kx, cw, left, W)):
            for y in range(254):
                for i in range(k):
                    c = tab[o_s + y] + i
                    if c < ext and 0 <= org + c < lim:
                        M[y, org + c] += wts[o_w + y * k + i]
        out[f] = torch.einsum("yh,chw,xw->cyx", Wy, im, Wx)
    return out


@pytest.mark.parametrize("name", ["a", "b", "c"])
def test_crop_table_matches_restated_crops(golden, name):
    """The host table (start indices, antialiased tap weights, zero fill, identity shortcut, center-crop offsets) gathers the
    crops of F.interpolate(antialias=True) in fp64; the tap weights are stored in fp32."""
    from mas_b200 import ops
    from face_common import prepare
    case = golden[name]
    img, rec = case_inputs(case)
    plan = ops.FacePlan(img.shape, rec.shape, case["boxes"])
    x = _crop_table_gather(plan, img, rec)
    assert tuple(x.shape) == case["crops_shape"]
    assert rel_err(x, prepare(img.double(), rec.double(), case["boxes"])) < 1e-7


@pytest.mark.parametrize("name", ["a", "b", "c"])
def test_restatement_reproduces_golden(golden, name):
    case = golden[name]
    m, _ = seeded_face_loss(case)
    img, rec = case_inputs(case)
    rec = rec.double().requires_grad_(case["drec"] is not None)
    x, feats, terms, loss = restated_loss(m, img.double(), rec, case["boxes"])
    c = case["crops"]
    assert tuple(x.shape) == case["crops_shape"]
    # the golden crops are the fp32 reference's: its separable fp32 resize is good to a few 1e-6 on the samples
    assert abs(float(x.norm()) - c["norm"]) <= 1e-6 * c["norm"] and rel_err(x.reshape(-1)[c["idx"]], c["val"]) < 1e-5
    for f, halves in zip(feats, case["features"]):
        for h, r in zip(f.chunk(2), halves):
            assert abs(float(h.norm()) - r["norm"]) <= 1e-5 * r["norm"]
            assert rel_err(h.reshape(-1)[r["idx"]], r["val"]) < 1e-5
    for t, r in zip(terms, case["terms"]):
        assert abs(float(t) - r) <= 1e-5 * abs(r)
    assert abs(float(loss) - case["loss"]) <= 1e-5 * case["loss"]
    if case["drec"] is not None:
        loss.backward()
        d = case["drec"]
        assert abs(float(rec.grad.norm()) - d["norm"]) <= 1e-5 * d["norm"]
        # sampled entries include small ones, where the fp32 reference's own rounding shows
        assert rel_err(rec.grad.reshape(-1)[d["idx"]], d["val"]) < 5e-5
