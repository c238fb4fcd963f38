"""VQBASE — drop-in for reference models/vqvae.py:8-39 over the sm_90a kernels in libmas_b200.so.

Same constructor/forward signatures and state_dict keys (348 entries for conf/img_config.yaml); parameters are
held by stock torch.nn holders created in the reference's order, so `torch.manual_seed(s)` gives identical
initial weights and checkpoints load in both directions.
"""
import torch
from torch import nn

from mas_b200 import ops

from .modules import Codebook, Conv2d, Decoder, Encoder


class QuantBatchNorm(nn.SyncBatchNorm):
    """nn.SyncBatchNorm(embed_dim) of vqvae.py:16: kernel-computed local sums + one NCCL all-reduce of 2*C numbers."""

    def forward(self, x):
        if self.training:
            if self.num_batches_tracked is not None:
                self.num_batches_tracked.add_(1)
            mom = self.momentum if self.momentum is not None else 1.0 / float(self.num_batches_tracked)
            return ops.BatchNormFn.apply(x, self.weight, self.bias, self.running_mean, self.running_var, mom, self.eps, True)
        return ops.batchnorm_eval(x, self.weight, self.bias, self.running_mean, self.running_var, self.eps)


class VQBASE(nn.Module):
    def __init__(self, ddconfig, n_embed, embed_dim, init_steps=2000, reservoir_size=2e5):
        # init_steps / reservoir_size defaults tolerate conf/seg_config.yaml, which omits them (SURVEY.md 3.5)
        super().__init__()
        ddconfig = dict(ddconfig)
        self.encoder = Encoder(**ddconfig)
        self.decoder = Decoder(**ddconfig)
        self.quantize = Codebook(n_embed, embed_dim, beta=0.25, init_steps=init_steps, reservoir_size=reservoir_size)
        self.quant_conv = nn.Sequential(Conv2d(ddconfig["z_channels"], embed_dim, 1), QuantBatchNorm(embed_dim))
        self.post_quant_conv = Conv2d(embed_dim, ddconfig["z_channels"], 1)

    def encode(self, x):
        """image [B,3,H,W] -> (quantised latent [B,embed_dim,h,w], codebook loss); vqvae.py:20-24."""
        z_q, codebook_loss, _indices = self.quantize(self.quant_conv(self.encoder(x)))
        return z_q, codebook_loss

    def decode(self, quant):
        """quantised latent -> reconstruction; vqvae.py:26-29."""
        return self.decoder(self.post_quant_conv(quant))

    def decode_code(self, code_b, shape=None):
        """Reference vqvae.py:31-34 calls a non-existent `embed_code`; implemented via get_codebook_entry.
        code_b: [B,h,w] (or [B,h*w] with `shape`=(B,h,w,C)) int64 indices."""
        if shape is None:
            b, h, w = code_b.shape
            shape = (b, h, w, self.quantize.codebook_dim)
        quant_b = self.quantize.get_codebook_entry(code_b.reshape(-1), shape)
        return self.decode(quant_b)

    def forward(self, input):
        """-> (dec, diff) exactly like vqvae.py:36-39 (train.py:84 unpacks this pair)."""
        z_q, diff = self.encode(input)
        return self.decode(z_q), diff
