"""LPIPS perceptual loss — drop-in for the reference's losses/lpips.py over the sm_90a kernels in libmas_b200.so.

Same classes (`LPIPS`, `VGG16`, `ScalingLayer`, `NetLinLayer`), constructor and state_dict as the reference, so `vgg.pth`
and checkpoints load in both directions, and `lpips_with_object.py`'s `from .lpips import LPIPS` subclasses this one.
The weights come from the same sources: torchvision's ImageNet VGG16 `features`, then the LPIPS checkpoint (`vgg16`,
`get_ckpt_path` and `load_checkpoint` are module-level so they can be replaced). forward() runs ops.LPIPSFn: no arithmetic
of the loss runs in PyTorch. The loss is evaluated with its parameters frozen and in eval mode, as loss_img.py builds it:
training-mode Dropout, weight gradients and double backward have no kernels and are refused."""
import os
import urllib.request

import torch
import torch.nn as nn

from mas_b200 import ops

URL_MAP = {
    "vgg_lpips": "https://heibox.uni-heidelberg.de/f/607503859c864bc1b30b/?dl=1"
}

# where the LPIPS head weights are looked for (and downloaded to when missing); MAS_LPIPS_CKPT overrides it
CKPT_MAP = {
    "vgg_lpips": os.environ.get("MAS_LPIPS_CKPT", os.path.join(os.path.expanduser("~"), ".cache", "make-a-scene", "vgg.pth"))
}


def vgg16(pretrained=True):
    """torchvision's VGG16 (ImageNet weights when pretrained); imported here so that replacing this factory needs no torchvision."""
    import torchvision
    return torchvision.models.vgg16(weights=torchvision.models.VGG16_Weights.IMAGENET1K_V1 if pretrained else None)


def get_ckpt_path(name, root=None):
    """Local path of the named checkpoint, downloaded first when it is missing."""
    if name not in URL_MAP:
        raise KeyError(name)
    path = CKPT_MAP[name]
    if not os.path.exists(path):
        os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
        print(f"Downloading {name} model from {URL_MAP[name]} to {path}")
        tmp = path + ".part"
        urllib.request.urlretrieve(URL_MAP[name], tmp)
        os.replace(tmp, path)
    return path


def load_checkpoint(path):
    return torch.load(path, map_location=torch.device("cpu"))


class ScalingLayer(nn.Module):
    def __init__(self):
        super().__init__()
        self.register_buffer("shift", torch.Tensor([-.030, -.088, -.188])[None, :, None, None])
        self.register_buffer("scale", torch.Tensor([.458, .448, .450])[None, :, None, None])

    def forward(self, x):
        raise RuntimeError("ScalingLayer runs inside LPIPS.forward (mas_lpips_prep)")


class NetLinLayer(nn.Module):
    def __init__(self, in_channels, out_channels=1):
        super().__init__()
        self.model = nn.Sequential(nn.Dropout(), nn.Conv2d(in_channels, out_channels, 1, 1, 0, bias=False))

    def forward(self, x):
        raise RuntimeError("NetLinLayer runs inside LPIPS.forward (mas_lpips_head_forward)")


class VGG16(nn.Module):
    """VGG16 `features[0:30]` split after relu1_2, relu2_2, relu3_3, relu4_3 and relu5_3; the stock layers hold the weights."""

    def __init__(self):
        super().__init__()
        features = vgg16(pretrained=True).features
        layers = [features[i] for i in range(30)]
        self.slice1 = nn.Sequential(*layers[0:4])
        self.slice2 = nn.Sequential(*layers[4:9])
        self.slice3 = nn.Sequential(*layers[9:16])
        self.slice4 = nn.Sequential(*layers[16:23])
        self.slice5 = nn.Sequential(*layers[23:30])
        for param in self.parameters():
            param.requires_grad = False

    def convs(self):
        """The 13 (weight, bias) pairs in layer order (checked against the structure the kernels implement)."""
        out = []
        for blk, s in enumerate((self.slice1, self.slice2, self.slice3, self.slice4, self.slice5)):
            mods = list(s)
            pooled = isinstance(mods[0], nn.MaxPool2d)
            if blk > 0 and not (pooled and mods[0].kernel_size in (2, (2, 2)) and mods[0].stride in (2, (2, 2))
                                and mods[0].padding in (0, (0, 0)) and not mods[0].ceil_mode):
                raise RuntimeError("LPIPS: VGG16 slice%d must start with MaxPool2d(2, 2)" % (blk + 1))
            body = mods[1:] if blk > 0 else mods
            if len(body) != 2 * ops.LPIPS_BLOCKS[blk]:
                raise RuntimeError("LPIPS: unexpected VGG16 slice%d layout" % (blk + 1))
            for conv, relu in zip(body[0::2], body[1::2]):
                if not (isinstance(conv, nn.Conv2d) and isinstance(relu, nn.ReLU) and conv.kernel_size == (3, 3)
                        and conv.padding == (1, 1) and conv.stride == (1, 1) and conv.dilation == (1, 1) and conv.groups == 1
                        and conv.bias is not None):
                    raise RuntimeError("LPIPS: VGG16 slice%d must hold Conv2d(3x3, padding 1) + ReLU pairs" % (blk + 1))
                out.append((conv.weight, conv.bias))
        return out

    def forward(self, x):
        raise RuntimeError("VGG16 runs inside LPIPS.forward")


class LPIPS(nn.Module):
    def __init__(self):
        super().__init__()
        self.scaling_layer = ScalingLayer()
        self.channels = [64, 128, 256, 512, 512]
        self.vgg = VGG16()
        self.lin0 = NetLinLayer(self.channels[0])
        self.lin1 = NetLinLayer(self.channels[1])
        self.lin2 = NetLinLayer(self.channels[2])
        self.lin3 = NetLinLayer(self.channels[3])
        self.lin4 = NetLinLayer(self.channels[4])
        self.load_from_pretrained()
        self.lins = [self.lin0, self.lin1, self.lin2, self.lin3, self.lin4]
        for param in self.parameters():
            param.requires_grad = False

    def load_from_pretrained(self, name="vgg_lpips"):
        self.load_state_dict(load_checkpoint(get_ckpt_path(name, "vgg_lpips")), strict=False)

    def forward(self, real_x, fake_x):
        """-> [B, 1, 1, 1] fp32: sum over relu1_2 .. relu5_3 of the spatial mean of lin((n(real) - n(fake))^2)."""
        self.check()
        lins = [lin.model[1].weight for lin in self.lins]
        keep = torch.is_grad_enabled() and (real_x.requires_grad or fake_x.requires_grad)
        return ops.LPIPSFn.apply(real_x, fake_x, self.scaling_layer.shift, self.scaling_layer.scale, self.vgg.convs(), lins,
                                 keep)

    def check(self):
        """Refuses what has no kernel: training-mode Dropout and trainable parameters."""
        if self.training:
            raise RuntimeError("LPIPS: Dropout(p=0.5) in training mode has no kernel; call .eval() on the loss "
                               "(as losses/loss_img.py does)")
        trainable = [n for n, p in self.named_parameters() if p.requires_grad]
        if trainable:
            raise RuntimeError("LPIPS computes no weight gradients; its parameters must have requires_grad=False "
                               "(got %s)" % ", ".join(trainable))
