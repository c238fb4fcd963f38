"""PatchGAN discriminator — drop-in for the reference's losses/discriminator.py:8-38 over the sm_90a kernels in
libmas_b200.so.

Same constructor, `self.model = nn.Sequential(...)` layout and 22-entry state_dict as the reference. The parameter holders
are stock nn.Conv2d / nn.BatchNorm2d subclasses (class names still contain "Conv" / "BatchNorm") created in the reference's
order, so `Discriminator().apply(weights_init)` under `torch.manual_seed(s)` gives bit-identical weights and checkpoints
load in both directions.  forward() runs each convolution with the LeakyReLU that follows it fused into its epilogue, and
each BatchNorm2d with its LeakyReLU in one pass; BatchNorm statistics are those of each call's own batch, as in the
reference."""
import torch.nn as nn

from mas_b200 import ops


def weights_init(m):
    classname = m.__class__.__name__
    if classname.find('Conv') != -1:
        nn.init.normal_(m.weight.data, 0.0, 0.02)
    elif classname.find('BatchNorm') != -1:
        nn.init.normal_(m.weight.data, 1.0, 0.02)
        nn.init.constant_(m.bias.data, 0)


class Conv2d(nn.Conv2d):
    """nn.Conv2d(cin, cout, 4, stride, 1) on mas_conv4x4 (+ a fused LeakyReLU(slope) when slope is given)."""

    def forward(self, x, slope=None):
        if self.kernel_size != (4, 4) or self.padding != (1, 1) or self.stride[0] != self.stride[1] or self.dilation != (1, 1) \
                or self.groups != 1 or self.stride[0] not in (1, 2):
            raise RuntimeError("losses.discriminator.Conv2d runs 4x4 kernels with padding 1 and stride 1 or 2 only")
        return ops.Conv4x4Fn.apply(x, self.weight, self.bias, self.stride[0], slope)


class BatchNorm2d(nn.BatchNorm2d):
    """nn.BatchNorm2d (plain: statistics of this call's batch) + a fused LeakyReLU(slope) (slope 1: none)."""

    def forward(self, x, slope=1.0):
        if self.training:
            if self.num_batches_tracked is not None:
                self.num_batches_tracked.add_(1)
            mom = self.momentum if self.momentum is not None else 1.0 / float(self.num_batches_tracked)
            return ops.BatchNormLReLUFn.apply(x, self.weight, self.bias, self.running_mean, self.running_var, mom, self.eps,
                                              slope)
        return ops.batchnorm_lrelu_eval(x, self.weight, self.bias, self.running_mean, self.running_var, self.eps, slope)


class Discriminator(nn.Module):
    def __init__(self, in_channels=3, num_filters_last=64, n_layers=3):
        super(Discriminator, self).__init__()

        layers = [Conv2d(in_channels, num_filters_last, 4, 2, 1), nn.LeakyReLU(0.2)]
        num_filters_mult = 1

        for i in range(1, n_layers + 1):
            num_filters_mult_last = num_filters_mult
            num_filters_mult = min(2 ** i, 8)
            layers += [
                Conv2d(num_filters_last * num_filters_mult_last, num_filters_last * num_filters_mult, 4,
                       2 if i < n_layers else 1, 1, bias=False),
                BatchNorm2d(num_filters_last * num_filters_mult),
                nn.LeakyReLU(0.2, True)
            ]

        layers.append(Conv2d(num_filters_last * num_filters_mult, 1, 4, 1, 1))
        self.model = nn.Sequential(*layers)

    def forward(self, x):
        """-> [B, 1, h, w] fp32 logits (an ordinary contiguous NCHW tensor)."""
        mods = list(self.model)
        i = 0
        while i < len(mods):
            m = mods[i]
            nxt = mods[i + 1] if i + 1 < len(mods) else None
            if isinstance(nxt, nn.LeakyReLU) and isinstance(m, (Conv2d, BatchNorm2d)):
                x = m(x, nxt.negative_slope)
                i += 2
            elif isinstance(m, (Conv2d, BatchNorm2d)):
                x = m(x)
                i += 1
            else:
                raise RuntimeError("Discriminator.forward: unexpected module %s" % type(m).__name__)
        return x.contiguous()
