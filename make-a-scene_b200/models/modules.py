"""Drop-in for reference models/modules.py (Encoder/Decoder/ResnetBlock/AttnBlock/Codebook ...) on sm_90a kernels.

Every class keeps the reference's name, constructor signature, attribute names and parameter shapes
(modules.py:35-240,337-369,451-528); forward passes run exclusively through libmas_b200.so
(mas_b200.ops). Activations travel between modules as channels-last tensors of logical shape [N,C,H,W];
the first convolution reads, and the last one writes, the caller's NCHW layout directly.
"""
import math

import torch
import torch.distributed as dist
import torch.nn as nn

from mas_b200 import _lib as L
from mas_b200 import ops


def nonlinearity(x):
    """swish, modules.py:35-37."""
    return ops.SiLUFn.apply(x)


class GroupNorm(torch.nn.GroupNorm):
    """torch.nn.GroupNorm holder whose forward runs the fused statistics/apply kernels."""

    def forward(self, x, silu=False):
        if self.num_groups != ops.GN_GROUPS or abs(self.eps - ops.GN_EPS) > 0 or not self.affine:
            raise RuntimeError("GroupNorm kernel is specialised to Normalize(): 32 groups, eps=1e-6, affine")
        return ops.GroupNormFn.apply(x, self.weight, self.bias, silu)


def Normalize(in_channels):
    """modules.py:40-41."""
    return GroupNorm(num_groups=32, num_channels=in_channels, eps=1e-6, affine=True)


class Swish(nn.Module):
    """modules.py:194-196."""

    def forward(self, x):
        return ops.SiLUFn.apply(x)


class Conv2d(torch.nn.Conv2d):
    """torch.nn.Conv2d parameter holder (identical default init) dispatching to the conv / GEMM kernels.
    Supported: 3x3 s1 p1, 1x1 s1 p0, and (through Downsample) 3x3 s2 p0 with the (0,1,0,1) zero pad."""

    out_nchw = False  # set on the decoder's last conv so that `dec` is a plain NCHW tensor like the reference's

    def forward(self, x, residual=None, mode=None):
        k, s, p = self.kernel_size, self.stride, self.padding
        if k == (1, 1) and s == (1, 1) and p == (0, 0) and residual is None:
            return ops.Conv1x1Fn.apply(x, self.weight, self.bias)
        if k == (3, 3):
            if mode is None:
                if s == (1, 1) and p == (1, 1):
                    mode = L.CONV_S1
                else:
                    raise RuntimeError("Conv2d 3x3 with stride %s padding %s has no kernel; use Downsample/Upsample" % (s, p))
            return ops.Conv3x3Fn.apply(x, self.weight, self.bias, residual, mode, self.out_nchw)
        raise RuntimeError("unsupported Conv2d configuration k=%s s=%s p=%s (no fallback path)" % (k, s, p))


class Upsample(nn.Module):
    """modules.py:44-59 — nearest x2 folded into the convolution's input gather (no 4x intermediate)."""

    def __init__(self, in_channels, with_conv):
        super().__init__()
        self.with_conv = with_conv
        if self.with_conv:
            self.conv = Conv2d(in_channels, in_channels, kernel_size=3, stride=1, padding=1)

    def forward(self, x):
        if not self.with_conv:
            raise RuntimeError("Upsample(with_conv=False) is never built by Encoder/Decoder and has no kernel")
        return self.conv(x, mode=L.CONV_UP)


class Downsample(nn.Module):
    """modules.py:62-81 — the (0,1,0,1) zero pad is handled by bounds in the stride-2 gather."""

    def __init__(self, in_channels, with_conv):
        super().__init__()
        self.with_conv = with_conv
        if self.with_conv:
            self.conv = Conv2d(in_channels, in_channels, kernel_size=3, stride=2, padding=0)

    def forward(self, x):
        if not self.with_conv:
            raise RuntimeError("Downsample(with_conv=False) is never built by Encoder/Decoder and has no kernel")
        if x.shape[2] % 2 or x.shape[3] % 2:
            raise RuntimeError("Downsample kernel needs even H and W")
        return self.conv(x, mode=L.CONV_S2)


class ResnetBlock(nn.Module):
    """modules.py:84-136."""

    def __init__(self, *, in_channels, out_channels=None, conv_shortcut=False, dropout):
        super().__init__()
        self.in_channels = in_channels
        out_channels = in_channels if out_channels is None else out_channels
        self.out_channels = out_channels
        self.use_conv_shortcut = conv_shortcut
        self.norm1 = Normalize(in_channels)
        self.conv1 = Conv2d(in_channels, out_channels, kernel_size=3, stride=1, padding=1)
        self.norm2 = Normalize(out_channels)
        self.dropout = torch.nn.Dropout(dropout)
        self.conv2 = Conv2d(out_channels, out_channels, kernel_size=3, stride=1, padding=1)
        if self.in_channels != self.out_channels:
            if self.use_conv_shortcut:
                self.conv_shortcut = Conv2d(in_channels, out_channels, kernel_size=3, stride=1, padding=1)
            else:
                self.nin_shortcut = Conv2d(in_channels, out_channels, kernel_size=1, stride=1, padding=0)

    def forward(self, x):
        if self.dropout.p != 0.0 and self.training:
            raise RuntimeError("dropout>0 is never used by the reference (modules.py:224) and has no kernel")
        if self.in_channels != self.out_channels and self.use_conv_shortcut:
            h = self.norm1(x, silu=True)
            h = self.conv1(h)
            h = self.norm2(h, silu=True)
            return self.conv2(h, residual=self.conv_shortcut(x))
        sc = self.nin_shortcut if self.in_channels != self.out_channels else None
        st = ops.take_stats(x)   # GroupNorm statistics emitted by the producing kernel's epilogue, if any
        # x produced by another ResnetBlock: its backward will read our dx through the TMA-fed data-gradient convolution, so
        # our GroupNorm backward also writes dx as an fp16 shadow (ops.gn_backward(shadow=True))
        from_res = bool(getattr(x, "_mas_res_out", False))
        out, mo, ro = ops.ResnetBlockFn.apply(x, st[0], st[1], self.norm1.weight, self.norm1.bias, self.conv1.weight,
                                              self.conv1.bias, self.norm2.weight, self.norm2.bias, self.conv2.weight,
                                              self.conv2.bias, None if sc is None else sc.weight, None if sc is None else sc.bias,
                                              from_res)
        out._mas_res_out = True
        return ops.attach_stats(out, mo, ro)


class AttnBlock(nn.Module):
    """modules.py:139-191."""

    def __init__(self, in_channels):
        super().__init__()
        self.in_channels = in_channels
        self.norm = Normalize(in_channels)
        self.q = Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.k = Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.v = Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)
        self.proj_out = Conv2d(in_channels, in_channels, kernel_size=1, stride=1, padding=0)

    def forward(self, x):
        st = ops.take_stats(x)
        out, mo, ro = ops.AttnBlockFn.apply(x, st[0], st[1], self.norm.weight, self.norm.bias, self.q.weight, self.q.bias,
                                            self.k.weight, self.k.bias, self.v.weight, self.v.bias, self.proj_out.weight,
                                            self.proj_out.bias)
        return ops.attach_stats(out, mo, ro)


def _run(model, x):
    """nn.Sequential forward with one peephole: (Normalize, Swish) pairs run as a single fused kernel."""
    mods = list(model)
    i = 0
    while i < len(mods):
        m = mods[i]
        if isinstance(m, GroupNorm) and i + 1 < len(mods) and isinstance(mods[i + 1], Swish):
            x = m(x, silu=True)
            i += 2
        else:
            x = m(x)
            i += 1
    return x


class Encoder(nn.Module):
    """modules.py:199-240. Stale taming keys (ch, ch_mult, out_ch, double_z, ...) are swallowed by **kwargs exactly
    like the reference does."""

    def __init__(self, in_channels=3, channels=[128, 128, 128, 256, 512, 512], attn_resolutions=[32], resolution=512,
                 dropout=0.0, num_res_blocks=2, z_channels=256, **kwargs):
        super().__init__()
        layers = [Conv2d(in_channels, channels[0], 3, 1, 1)]
        for i in range(len(channels) - 1):
            in_channels = channels[i]
            out_channels = channels[i + 1]
            for j in range(num_res_blocks):
                layers.append(ResnetBlock(in_channels=in_channels, out_channels=out_channels, dropout=0.0))
                in_channels = out_channels
                if resolution in attn_resolutions:
                    layers.append(AttnBlock(in_channels))
            if i < len(channels) - 2:
                layers.append(Downsample(channels[i + 1], with_conv=True))
                resolution //= 2
        layers.append(ResnetBlock(in_channels=channels[-1], out_channels=channels[-1], dropout=0.0))
        layers.append(AttnBlock(channels[-1]))
        layers.append(ResnetBlock(in_channels=channels[-1], out_channels=channels[-1], dropout=0.0))
        layers.append(Normalize(channels[-1]))
        layers.append(Swish())
        layers.append(Conv2d(channels[-1], z_channels, 3, 1, 1))
        self.model = nn.Sequential(*layers)

    def forward(self, x):
        return _run(self.model, x)


class Decoder(nn.Module):
    """modules.py:337-369. Bug-compatible with the reference: the stale taming key `out_ch` (conf/seg_config.yaml) is
    swallowed by **kwargs and IGNORED, so the output width is `out_channels` (default 3) — SURVEY.md 3.5. Pass
    out_channels explicitly for the 159-channel segmentation decoder."""

    def __init__(self, out_channels=3, channels=[128, 128, 128, 256, 512, 512], attn_resolutions=[32], resolution=512,
                 dropout=0.0, num_res_blocks=2, z_channels=256, **kwargs):
        super().__init__()
        ch_mult = channels[1:]
        num_resolutions = len(ch_mult)
        block_in = ch_mult[num_resolutions - 1]
        curr_res = resolution // 2 ** (num_resolutions - 1)
        layers = [Conv2d(z_channels, block_in, kernel_size=3, stride=1, padding=1),
                  ResnetBlock(in_channels=block_in, out_channels=block_in, dropout=0.0),
                  AttnBlock(block_in),
                  ResnetBlock(in_channels=block_in, out_channels=block_in, dropout=0.0)]
        for i in reversed(range(num_resolutions)):
            block_out = ch_mult[i]
            for i_block in range(num_res_blocks + 1):
                layers.append(ResnetBlock(in_channels=block_in, out_channels=block_out, dropout=0.0))
                block_in = block_out
                if curr_res in attn_resolutions:
                    layers.append(AttnBlock(block_in))
            if i > 0:
                layers.append(Upsample(block_in, with_conv=True))
            curr_res = curr_res * 2
        layers.append(Normalize(block_in))
        layers.append(Swish())
        last = Conv2d(block_in, out_channels, kernel_size=3, stride=1, padding=1)
        last.out_nchw = True
        layers.append(last)
        self.model = nn.Sequential(*layers)

    def forward(self, x):
        return _run(self.model, x)


class Codebook(nn.Module):
    """modules.py:451-528 — vector quantiser with reservoir sampling and k-means re-initialisation.
    The distance/argmin/gather/loss/straight-through chain (modules.py:501-515) is one CUDA kernel."""

    def __init__(self, codebook_size, codebook_dim, beta, init_steps=2000, reservoir_size=2e5):
        super().__init__()
        self.codebook_size = codebook_size
        self.codebook_dim = codebook_dim
        self.beta = beta
        self.embedding = nn.Embedding(self.codebook_size, self.codebook_dim)
        self.embedding.weight.data.uniform_(-1.0 / self.codebook_size, 1.0 / self.codebook_size)
        self.q_start_collect, self.q_init, self.q_re_end, self.q_re_step = init_steps, init_steps * 3, init_steps * 30, init_steps // 2
        self.q_counter = 0
        self.reservoir_size = int(reservoir_size)
        self.reservoir = None

    # -- rare training-time side paths (host logic, outside the steady state: modules.py:474-499) -------------
    def _collect(self, z):
        b = z.shape[0]
        zf = z.detach().permute(0, 2, 3, 1).reshape(b, -1, self.codebook_dim)
        z_new = zf[:, torch.randperm(zf.size(1), device=zf.device)][:, :10].reshape(-1, self.codebook_dim)
        self.reservoir = z_new if self.reservoir is None else torch.cat([self.reservoir, z_new], dim=0)
        self.reservoir = self.reservoir[torch.randperm(self.reservoir.size(0), device=z.device)[:self.reservoir_size]].detach()

    def _kmeans_reinit(self, iters=20, seed=0):
        """Replaces fast_pytorch_kmeans.KMeans (absent third-party, modules.py:489-499): Lloyd iterations whose
        assignment step is the VQ kernel; seeded and identical on all ranks (the reference's is neither)."""
        world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        res = self.reservoir
        if world > 1:
            parts = [torch.zeros_like(res) for _ in range(world)]
            dist.all_gather(parts, res.clone())
            res = torch.cat(parts, dim=0)
        g = torch.Generator(device="cpu").manual_seed(seed + self.q_counter)
        n = res.shape[0]
        pick = torch.randperm(n, generator=g)[:self.codebook_size].to(res.device)
        cent = res[pick].clone()
        if cent.shape[0] < self.codebook_size:
            cent = torch.cat([cent, self.embedding.weight.data[cent.shape[0]:]], 0)
        rows = res.contiguous().view(1, n, 1, self.codebook_dim).permute(0, 3, 1, 2)  # [1,D,n,1] channels-last view
        resc = res.contiguous()
        shift = torch.empty(1, dtype=torch.float32, device=res.device)
        ws = L.workspace(L.query("mas_kmeans_ws_bytes", cent.shape[0], self.codebook_dim), res.device)
        for _ in range(iters):
            _, _, idx = ops.VQFn.apply(rows, cent, 0.0)               # assignment: the VQ kernel
            new = torch.empty_like(cent)                                # update: segmented mean + centre shift, one call
            L.call("mas_kmeans_update", resc, idx, n, cent.shape[0], self.codebook_dim, cent, new, shift, ws, ws.numel())
            cent = new
            if float(shift) < 1e-4:
                break
        self.embedding.weight.data = cent.detach()

    def forward(self, z):
        if self.training:
            self.q_counter += 1
            if self.q_counter > self.q_start_collect:
                if getattr(self, "defer_collect", False):   # under a captured step (mas_b200.graph): sampled after the replay
                    self._deferred_z = z.detach()
                else:
                    self._collect(z)
            if self.q_counter < self.q_init:
                return ops.nhwc(z), z.new_tensor(0), None  # warm-up bypass, modules.py:482-484
            if self.q_init <= self.q_counter < self.q_re_end:
                if (self.q_counter - self.q_init) % self.q_re_step == 0 or self.q_counter == self.q_init + self.q_re_end - 1:
                    print("Updating codebook from reservoir.")
                    self._kmeans_reinit()
        z_q, loss, min_encoding_indices = ops.VQFn.apply(z, self.embedding.weight, self.beta)
        return z_q, loss, min_encoding_indices

    def get_codebook_entry(self, indices, shape):
        """modules.py:519-528."""
        z_q = ops.vq_gather(self.embedding.weight.detach(), indices)
        if shape is not None:
            z_q = z_q.view(shape).permute(0, 3, 1, 2)  # NHWC memory, NCHW logical (values identical to the reference)
        return z_q
