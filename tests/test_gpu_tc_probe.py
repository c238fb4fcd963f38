"""GPU: pins the wgmma operand conventions (shared-memory descriptor majorness, A from registers) with a one-MMA probe.
Descriptors are built in the sm_100 encoding: the probe drops its version bits; the swizzle codes 2 / 4 / 6 at bit 61 are the
sm_90 128 / 64 / 32-byte codes at bit 62, and bit 16 of the instruction descriptor selects an MN-major (transposed) B."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("a_src,b_layout", [(0, 0), (1, 0), (0, 1), (1, 1), (0, 2), (1, 2)])
def test_single_mma_conventions(a_src, b_layout):
    from mas_b200 import _lib as L
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(5)
    A = torch.randn(128, 8, generator=g).to(dev)
    B = torch.randn(32, 8, generator=g).to(dev)
    D = torch.full((128, 32), float("nan"), device=dev)
    L.call("mas_tc_probe", A, B, D, a_src, b_layout, 0, 0, 0)
    ref = A.double() @ B.double().t()
    err = float((D.double() - ref).norm() / ref.norm())
    print(f"probe a_src={a_src} b_layout={b_layout}: rel err {err:.3e} D[0,:4]={D[0,:4].tolist()} ref={ref[0,:4].tolist()}")
    if b_layout == 0:
        assert err < 2e-3, (a_src, b_layout, err)   # K-major B; A from smem (SS) and from registers (RS) both work
    else:
        # wgmma transposes 16-bit operands only: an MN-major TF32 image is read as K-major and the product is wrong, so the
        # production kernels keep every TF32 smem operand K-major (see wgrad_tc's transposed halo copies)
        assert err > 0.5


@pytest.mark.parametrize("b_layout", [0, 1, 2])
def test_reveal_b_addressing(b_layout):
    """A = selector (row m picks k = m % 8), B region = its own word index: D[k][n] is the shared-memory word the
    tensor core reads for element (n, k) of B under the given descriptor convention."""
    from mas_b200 import _lib as L
    dev = torch.device("cuda:0")
    A = torch.zeros(128, 8)
    for m in range(128):
        A[m, m % 8] = 1.0
    D = torch.full((128, 32), float("nan"), device=dev)
    L.call("mas_tc_probe", A.to(dev), torch.zeros(32, 8, device=dev), D, 0, 10 + b_layout, 0, 0, 0)
    off = D[:8].t().cpu().long()          # [n][k]
    print(f"REVEAL b_layout={b_layout}")
    for n in list(range(0, 10)) + [16, 31]:
        print("  n=%2d:" % n, off[n].tolist())


def _desc(lbo, sbo, layout_type, base_off=0):
    return ((lbo >> 4) << 16) | ((sbo >> 4) << 32) | (1 << 46) | (base_off << 49) | (layout_type << 61)


def _idesc(n, b_mn):
    return (1 << 4) | (2 << 7) | (2 << 10) | ((1 << 16) if b_mn else 0) | ((n >> 3) << 17) | ((128 >> 4) << 24)


RAW = [  # name, lbo, sbo, layout_type, b_mn, start_off, base_off
    ("K-major none (control)", 512, 128, 0, 0, 0, 0),
    ("MN none lbo160 sbo576", 160, 576, 0, 1, 0, 0),
    ("MN sw128 lbo1024 sbo1024", 1024, 1024, 2, 1, 0, 0),
    ("MN sw128 lbo4096 sbo1024", 4096, 1024, 2, 1, 0, 0),
    ("MN sw128 start+128", 4096, 1024, 2, 1, 128, 0),
    ("MN sw128 start+128 base1", 4096, 1024, 2, 1, 128, 1),
    ("MN sw128 start+256", 4096, 1024, 2, 1, 256, 0),
    ("MN sw64 lbo512 sbo512", 512, 512, 4, 1, 0, 0),
    ("MN sw32 lbo256 sbo256", 256, 256, 6, 1, 0, 0),
    ("K sw128 sbo1024", 16, 1024, 2, 0, 0, 0),
    ("K sw128 start+128", 16, 1024, 2, 0, 128, 0),
    ("K sw128 start+128 base1", 16, 1024, 2, 0, 128, 1),
    ("K sw128 start+32 (k advance)", 16, 1024, 2, 0, 32, 0),
]


@pytest.mark.parametrize("case", RAW, ids=[c[0] for c in RAW])
def test_reveal_raw(case):
    from mas_b200 import _lib as L
    name, lbo, sbo, lt, b_mn, off, base = case
    dev = torch.device("cuda:0")
    A = torch.zeros(128, 8)
    for m in range(128):
        A[m, m % 8] = 1.0
    D = torch.full((128, 32), float("nan"), device=dev)
    L.call("mas_tc_probe", A.to(dev), torch.zeros(32, 8, device=dev), D, 0, 99, _desc(lbo, sbo, lt, base), _idesc(32, b_mn), off)
    o = D[:8].t().cpu().long()
    print(f"RAW {name}")
    for n in list(range(0, 9)) + [12, 16, 31]:
        print("  n=%2d:" % n, o[n].tolist())


def _idesc16(n, b_mn, a_mn=0):
    return (1 << 4) | ((1 << 15) if a_mn else 0) | ((1 << 16) if b_mn else 0) | ((n >> 3) << 17) | ((128 >> 4) << 24)


RAW16 = [  # name, lbo, sbo, layout_type, b_mn, start_off
    ("f16 K-major none (control)", 512, 128, 0, 0, 0),
    ("f16 MN none lbo512 sbo128", 512, 128, 0, 1, 0),
    ("f16 MN none lbo128 sbo512", 128, 512, 0, 1, 0),
    ("f16 MN none lbo256 sbo128", 256, 128, 0, 1, 0),
    ("f16 MN none lbo128 sbo256", 128, 256, 0, 1, 0),
    ("f16 MN none lbo1024 sbo256", 1024, 256, 0, 1, 0),
    ("f16 MN none lbo256 sbo1024", 256, 1024, 0, 1, 0),
    ("f16 MN none start+16", 512, 128, 0, 1, 16),
    ("f16 MN sw128 lbo1024 sbo1024", 1024, 1024, 2, 1, 0),
]


@pytest.mark.parametrize("case", RAW16, ids=[c[0] for c in RAW16])
def test_reveal_raw_f16(case):
    """fp16 wgmma shared-memory operand addressing under MN-major / K-major descriptors (prints the half index read for each
    (n, k)); the K-major control must reproduce the layout the production kernels rely on: index = (k/8)*LBO/2 + n*8 + k%8."""
    from mas_b200 import _lib as L
    name, lbo, sbo, lt, b_mn, off = case
    dev = torch.device("cuda:0")
    D = torch.full((128, 32), float("nan"), device=dev)
    L.call("mas_tc_probe16", D, _desc(lbo, sbo, lt), _idesc16(32, b_mn), off)
    o = D[:16].t().cpu().long()           # [n][k]
    print(f"RAW16 {name}")
    for n in list(range(0, 10)) + [15, 16, 17, 31]:
        print("  n=%2d:" % n, o[n].tolist())
    if not b_mn:
        want = torch.tensor([[(k // 8) * (lbo // 2) + n * 8 + (k % 8) for k in range(16)] for n in range(32)])
        assert torch.equal(o, want)
