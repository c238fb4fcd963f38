"""VQBASE — drop-in for reference models/vqvae.py:8-39 over the sm_90a kernels in libmas_b200.so.

Same constructor/forward signatures and state_dict keys (348 entries for conf/img_config.yaml); parameters are
held by stock torch.nn holders created in the reference's order, so `torch.manual_seed(s)` gives identical
initial weights and checkpoints load in both directions.
"""
import torch
from torch import nn

from mas_b200 import ops, scene

from .modules import Codebook, Conv2d, Decoder, Downsample, Encoder


def _kernel_device(t):
    """Whether t lives where the kernels run."""
    return t.is_cuda


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

    def encode_code(self, x):
        """Codebook indices of an input: the counterpart of decode_code, for tokenizing images and scene maps for the token
        transformer (MakeAScene's img_tokens / seg_tokens are encode_code(x).flatten(1)).

        x: an fp32 image batch [B, in_channels, H, W], a dense fp32 scene map [B, 159, H, W] or a compact scene map uint8
        [B, 4, H, W] (mas_b200.scene; only when conv_in takes 159 channels), a CUDA tensor on the model's device, H and W
        multiples of the encoder's downsampling factor f = 2^(len(channels) - 2).
        Returns int64 [B, H/f, W/f], row-major: flatten(1) puts position (i, j) at t = i * w + j, which is where MakeAScene
        adds row embedding i and column embedding j, and decode_code(tokens) is the inverse.

        Always the eval-mode encoding, whatever the module's mode: encoder -> quant_conv[0] -> BatchNorm with the running
        statistics -> codebook arg-min (the forward's kernels). Codebook.forward and QuantBatchNorm.forward are not called,
        so nothing changes: no step counter, reservoir, k-means re-initialisation, running statistics or collective, and the
        module's mode is left alone. No autograd graph is recorded, even under torch.enable_grad(). Raises ValueError on a
        tensor off the model's device or not on CUDA, a wrong dtype or channel count, or H / W off the downsampling factor."""
        conv_in = self.encoder.model[0]
        dev = conv_in.weight.device
        if not isinstance(x, torch.Tensor) or x.dim() != 4:
            raise ValueError("encode_code expects a 4-D [B, C, H, W] tensor, got %s"
                             % (str(tuple(x.shape)) if isinstance(x, torch.Tensor) else type(x).__name__))
        if not _kernel_device(x) or x.device != dev:
            raise ValueError("encode_code needs a CUDA tensor on the model's device (%s), got one on %s" % (dev, x.device))
        b, c, h, w = x.shape
        if x.dtype == torch.uint8:
            if conv_in.in_channels != scene.CHANNELS or c != scene.PLANES:
                raise ValueError("a uint8 input is a compact scene map [B, %d, H, W] for a model whose conv_in takes %d "
                                 "channels; got shape %s for conv_in with %d" % (scene.PLANES, scene.CHANNELS, tuple(x.shape),
                                                                                 conv_in.in_channels))
        elif x.dtype != torch.float32:
            raise ValueError("encode_code takes float32 images / scene maps or uint8 compact scene maps, got %s" % x.dtype)
        elif c != conv_in.in_channels:
            raise ValueError("expected %d input channels (conv_in), got shape %s" % (conv_in.in_channels, tuple(x.shape)))
        f = 2 ** sum(isinstance(m, Downsample) for m in self.encoder.model)
        if b == 0 or h == 0 or w == 0 or h % f or w % f:
            raise ValueError("encode_code needs a non-empty batch with H and W multiples of %d, got shape %s" % (f, tuple(x.shape)))
        bn = self.quant_conv[1]
        with torch.no_grad():
            z = self.quant_conv[0](self.encoder(x))
            z = ops.batchnorm_eval(z, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.eps)
            _, _, idx = ops.VQFn.apply(z, self.quantize.embedding.weight, self.quantize.beta)
        return idx.view(b, h // f, w // f)

    def decode_scene(self, code_b):
        """Seg tokens -> the compact scene map they stand for: scene.decode(decode_code(code_b)), uint8 [B, 4, H, W] on the
        model's device (mas_b200.scene: 1 + the argmax of each one-hot group where its maximum logit is > 0, else 0; edges 0 / 1).
        The counterpart of encode_code for a VQ-SEG model: decode_scene(encode_code(labels)) is its round trip, and
        scene.iou(scene.confusion(decode_scene(encode_code(labels)), labels)) its quality.

        code_b: int64 [B, h, w] codebook indices on the model's device.  Only for a model whose decoder's last convolution has
        159 outputs.  The decoder has no mode-dependent layer, so this is the eval-mode decoding in either mode; nothing of the
        module changes and no autograd graph is recorded.  Raises ValueError on another model, a tensor off the model's
        device or not [B, h, w] int64."""
        conv_out = self.decoder.model[-1]
        dev = conv_out.weight.device
        if conv_out.out_channels != scene.CHANNELS:
            raise ValueError("decode_scene needs a VQ-SEG model (decoder output %d channels), this one has %d"
                             % (scene.CHANNELS, conv_out.out_channels))
        if not isinstance(code_b, torch.Tensor) or code_b.dim() != 3 or code_b.dtype != torch.int64 or 0 in code_b.shape:
            raise ValueError("decode_scene expects int64 tokens [B, h, w], got %s" % (
                "%s %s" % (tuple(code_b.shape), code_b.dtype) if isinstance(code_b, torch.Tensor) else type(code_b).__name__))
        if not _kernel_device(code_b) or code_b.device != dev:
            raise ValueError("decode_scene needs a CUDA tensor on the model's device (%s), got one on %s" % (dev, code_b.device))
        f = 2 ** sum(isinstance(m, Downsample) for m in self.encoder.model)
        b, h, w = code_b.shape
        if b > 65535 or h * f > 65535:
            raise ValueError("decode_scene needs B and H * %d at most 65535, got tokens of shape %s" % (f, tuple(code_b.shape)))
        with torch.no_grad():
            return scene.decode(self.decode_code(code_b))

    def forward(self, input):
        """-> (dec, diff) exactly like vqvae.py:36-39 (train.py:84 unpacks this pair)."""
        z_q, diff = self.encode(input)
        return self.decode(z_q), diff
