"""Writes tests/golden/encode_code.pt from the REAL reference VQBASE (models/ of a reference checkout), on the CPU in fp32:

    python tools/make_golden_encode_code.py --reference <reference checkout>

The reference imports the absent third-party fast_pytorch_kmeans; it is stubbed the way oracle/make_golden.py stubs it (the
k-means branch only runs in train mode, and every module here runs in eval mode). No weights are stored: they come from
torch.manual_seed and the constructors, which build the drop-in's parameters in the same order.

Two cases at batch 2, 256 x 256:
  img  the img_config model, seeded as for vqbase_img_256.pt, on a seeded image batch;
  seg  the seg_config model (out_channels=159) on a dense scene map expanded from seeded label planes (mas_b200.scene
       layout), so the compact map of the same input is known.
In both, quant_conv[1]'s running statistics are set from another seeded batch (its pre-BatchNorm latents: mean, and
variance x 1.5), and the codebook is spread the way the k-means re-initialisation leaves it: row k is base[k % NBASE] plus
N(0, SIGMA^2) noise, where base holds NBASE of the reference's own eval latents of that other batch. The default +-1/K
init would put every code near the origin. base, the running statistics and the noise seed are stored; codebook() rebuilds
the codebook bit for bit on the CPU.

Recorded per case: fp64 (sum, abs-sum) of every initial parameter; the eval latent after BatchNorm (norm and a strided
sample); the code indices [B, 16, 16]; decode(get_codebook_entry(idx)) (norm and a strided sample) - the reference's own
decode_code calls a method its Codebook does not have.
"""
import argparse
import hashlib
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "encode_code.pt")
IMG = dict(z_channels=256, in_channels=3, out_channels=3, channels=[128, 128, 128, 256, 512, 512], num_res_blocks=2,
           resolution=512, attn_resolutions=[32], dropout=0.0)
# conf/seg_config.yaml's model block (stale taming keys included; `channels` is absent there, so the default applies) with
# the decoder's width given explicitly: the reference's Decoder ignores `out_ch`
SEG = dict(double_z=False, z_channels=256, resolution=256, in_channels=159, out_ch=159, ch=128, ch_mult=[1, 1, 2, 2, 4],
           num_res_blocks=2, attn_resolutions=[16], dropout=0.0, out_channels=159)
CASES = {"img": dict(ddconfig=IMG, n_embed=8192, embed_dim=256, init_steps=3000, reservoir_size=12500, weight_seed=0,
                     x_seed=31, other_seed=32, noise_seed=33),
         "seg": dict(ddconfig=SEG, n_embed=1024, embed_dim=256, init_steps=2000, reservoir_size=200000, weight_seed=1,
                     x_seed=41, other_seed=42, noise_seed=43)}
BATCH, SIZE = 2, 256
NBASE, SIGMA = 128, 0.3
NSAMP = 8192


def labels(seed, n=BATCH, size=SIZE, cell=8):
    """Seeded compact scene map uint8 [n, 4, size, size] (mas_b200.scene planes): label regions of cell x cell pixels."""
    g = torch.Generator().manual_seed(seed)
    s = size // cell
    lab = torch.stack([torch.randint(0, 134, (n, s, s), generator=g), torch.randint(0, 21, (n, s, s), generator=g),
                       torch.randint(0, 6, (n, s, s), generator=g), torch.randint(0, 3, (n, s, s), generator=g)], 1)
    return lab.repeat_interleave(cell, 2).repeat_interleave(cell, 3).to(torch.uint8).contiguous()


def dense_map(lab):
    """Compact planes [n, 4, H, W] -> the dense [n, 159, H, W] fp32 map load_segmentation builds from the same labels."""
    lab = lab.long()
    seg = torch.cat([F.one_hot(lab[:, 0], 134)[..., 1:], F.one_hot(lab[:, 1], 21)[..., 1:], F.one_hot(lab[:, 2], 6)[..., 1:],
                     lab[:, 3, :, :, None]], -1)
    return seg.float().permute(0, 3, 1, 2).contiguous()


def inputs(name, seed):
    """The case's input batch for `seed` (x_seed: the recorded batch; other_seed: the batch the statistics and codebook come
    from). img: fp32 images in [-1, 1]; seg: the compact planes (the dense map is dense_map of them)."""
    if name == "img":
        return torch.rand(BATCH, 3, SIZE, SIZE, generator=torch.Generator().manual_seed(seed)) * 2 - 1
    return labels(seed)


def codebook(base, n_embed, noise_seed):
    """Row k = base[k % len(base)] + SIGMA * N(0, 1), from a CPU generator."""
    noise = torch.randn(n_embed, base.shape[1], generator=torch.Generator().manual_seed(noise_seed))
    return base[torch.arange(n_embed) % base.shape[0]] + SIGMA * noise


def sha(t):
    return hashlib.sha256(t.detach().contiguous().numpy().tobytes()).hexdigest()


def sample(t):
    f = t.detach().reshape(-1)
    stride = max(1, f.numel() // NSAMP) | 1          # odd: coprime to the power-of-two tile sizes
    return {"val": f[::stride].clone(), "stride": stride, "norm": float(f.double().norm()), "shape": tuple(t.shape)}


def latent(m, x):
    """Eval-mode latent after quant_conv (BatchNorm with the running statistics)."""
    return m.quant_conv(m.encoder(x))


def run_case(ref_models, name, ddconfig, n_embed, embed_dim, init_steps, reservoir_size, weight_seed, x_seed, other_seed,
             noise_seed):
    torch.manual_seed(weight_seed)
    m = ref_models.VQBASE(ddconfig, n_embed, embed_dim, init_steps, reservoir_size).eval()
    checks = {k: (float(p.detach().double().sum()), float(p.detach().double().abs().sum())) for k, p in m.named_parameters()}
    feed = (lambda lab: dense_map(lab)) if name == "seg" else (lambda t: t)
    bn = m.quant_conv[1]
    with torch.no_grad():
        pre = m.quant_conv[0](m.encoder(feed(inputs(name, other_seed))))
        bn.running_mean.copy_(pre.mean((0, 2, 3)))
        bn.running_var.copy_(pre.var((0, 2, 3)) * 1.5)
        lat_other = bn(pre).permute(0, 2, 3, 1).reshape(-1, embed_dim)
        base = lat_other[torch.randperm(lat_other.shape[0], generator=torch.Generator().manual_seed(noise_seed))[:NBASE]].clone()
        m.quantize.embedding.weight.copy_(codebook(base, n_embed, noise_seed))
        x = inputs(name, x_seed)
        z = latent(m, feed(x))
        _, _, idx = m.quantize(z)
        b, _, h, w = z.shape
        dec = m.decode(m.quantize.get_codebook_entry(idx, (b, h, w, embed_dim)))
    return {"n_embed": n_embed, "embed_dim": embed_dim, "init_steps": init_steps, "reservoir_size": reservoir_size,
            "weight_seed": weight_seed, "x_seed": x_seed, "noise_seed": noise_seed, "input_sha256": sha(x),
            "param_checks": checks, "running_mean": bn.running_mean.clone(), "running_var": bn.running_var.clone(),
            "base": base, "codebook_sha256": sha(m.quantize.embedding.weight), "latent": sample(z),
            "idx": idx.view(b, h, w).clone(), "dec": sample(dec)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", required=True, help="root of a reference checkout (holds models/)")
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    from oracle import make_golden
    make_golden.REF = os.path.abspath(a.reference)
    ref_models = make_golden.load_reference()[0]
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    out = {"batch": BATCH, "size": SIZE, "nbase": NBASE, "sigma": SIGMA}
    for name, kw in CASES.items():
        out[name] = dict(run_case(ref_models, name, **kw), ddconfig=kw["ddconfig"])
        print(name, "latent norm %.4f" % out[name]["latent"]["norm"], "distinct codes", int(out[name]["idx"].unique().numel()),
              "dec norm %.4f" % out[name]["dec"]["norm"])
    torch.save(out, OUT)
    print("wrote", OUT, "%.1f KiB" % (os.path.getsize(OUT) / 1024))


if __name__ == "__main__":
    main()
