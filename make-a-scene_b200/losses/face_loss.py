"""VGGFace2 face loss - drop-in for the reference's losses/face_loss.py over the sm_90a kernels in libmas_b200.so.

Same classes (`FaceLoss`, `Bottleneck`), constructor and state_dict (318 keys) as the reference, so its weight file and
checkpoints load in both directions, and loss_img.py's `from .face_loss import FaceLoss` picks this one up. The weights come
from `WEIGHTS` (the MAS_FACE_LOSS_WEIGHTS environment variable, else the reference's path) through `load_weights`, both
module-level so they can be replaced; torchvision is not needed. forward() runs ops.FaceLossFn: crops, resize, the ResNet-50
and the L1 taps all run on the kernels. The loss is evaluated with frozen parameters in eval mode, as loss_img.py builds
it: training-mode BatchNorm, weight gradients and double backward have no kernels and are refused."""
import os

import torch
import torch.nn as nn

from mas_b200 import ops

__all__ = ['FaceLoss']

# the weight file the constructor loads (strict=False); MAS_FACE_LOSS_WEIGHTS overrides the reference's location
WEIGHTS = os.environ.get("MAS_FACE_LOSS_WEIGHTS", "/home/ubuntu/Make-A-Scene/losses/face_loss_weights.pt")


def load_weights(path):
    """The state dict FaceLoss() loads from `path`."""
    if not os.path.exists(path):
        raise FileNotFoundError("FaceLoss weights not found at %r; point MAS_FACE_LOSS_WEIGHTS at the VGGFace2 ResNet-50 "
                                "weight file" % path)
    return torch.load(path, map_location="cpu")


def conv3x3(in_planes, out_planes, stride=1):
    """3x3 convolution with padding"""
    return nn.Conv2d(in_planes, out_planes, kernel_size=3, stride=stride, padding=1, bias=False)


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, kernel_size=1, stride=stride, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, kernel_size=3, stride=1, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, kernel_size=1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = downsample
        self.stride = stride

    def forward(self, x):
        raise RuntimeError("Bottleneck runs inside FaceLoss.forward (ops.FaceLossFn)")


class FaceLoss(nn.Module):
    def __init__(self):
        super().__init__()
        layers = [3, 4, 6, 3]
        self.inplanes = 64
        self.alphas = [0.1, 0.25 * 0.01, 0.25 * 0.1, 0.25 * 0.2, 0.25 * 0.02]

        self.conv1 = nn.Conv2d(3, 64, kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=0, ceil_mode=True)

        self.layer1 = self._make_layer(Bottleneck, 64, layers[0])
        self.layer2 = self._make_layer(Bottleneck, 128, layers[1], stride=2)
        self.layer3 = self._make_layer(Bottleneck, 256, layers[2], stride=2)
        self.layer4 = self._make_layer(Bottleneck, 512, layers[3], stride=2)

        self.channels = [64, 256, 512, 1024, 2048]

        self.load_state_dict(load_weights(WEIGHTS), strict=False)

        for param in self.parameters():
            param.requires_grad = False
        self.eval()

    def _make_layer(self, block, planes, blocks, stride=1):
        downsample = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            downsample = nn.Sequential(
                nn.Conv2d(self.inplanes, planes * block.expansion, kernel_size=1, stride=stride, bias=False),
                nn.BatchNorm2d(planes * block.expansion),
            )
        layers = [block(self.inplanes, planes, stride, downsample)]
        self.inplanes = planes * block.expansion
        for _ in range(1, blocks):
            layers.append(block(self.inplanes, planes))
        return nn.Sequential(*layers)

    def _check(self):
        if self.training:
            raise RuntimeError("FaceLoss: BatchNorm in training mode (batch statistics) has no kernel; call .eval() on the "
                               "loss (the constructor does)")
        trainable = [n for n, p in self.named_parameters() if p.requires_grad]
        if trainable:
            raise RuntimeError("FaceLoss computes no weight gradients; its parameters must have requires_grad=False "
                               "(got %s)" % ", ".join(trainable))

    def forward(self, img, rec, bbox):
        """sum over the five taps of alpha_l * mean_{c,h,w} sum_pairs |a - b| over the first six stacked crops
        [gt_1 .. gt_n, gen_1 .. gen_n], first half against second half -> 0-dim fp32 tensor (img.new_tensor(0) without faces)."""
        self._check()
        plan = ops.FacePlan(img.shape, rec.shape, bbox)
        if plan.F == 0:
            return img.new_tensor(0)
        if 1 not in plan.sides():
            rec = rec.detach()          # only gt crops run (n >= 6): nothing depends on rec
        return ops.FaceLossFn.apply(img, rec, plan, ops.face_params(self))

    @torch.no_grad()
    def features(self, img, rec, bbox):
        """(crops [F, 3, 254, 254], the five features, the five level terms, loss) of the crops forward() runs (None without
        faces); tensors are channels-last."""
        self._check()
        plan = ops.FacePlan(img.shape, rec.shape, bbox)
        if plan.F == 0:
            return None
        r = ops.face_forward_raw(img, rec, plan, ops.face_params(self))
        return r["crops"], r["feats"], r["terms"], r["loss"]

    @torch.no_grad()
    def prepare_faces(self, imgs, recs, bboxes):
        """All stacked crops [gt_1 .. gt_n, gen_1 .. gen_n] as [2n, 3, 254, 254] (None without boxes), gathered by the same
        kernel as forward(). Unlike the reference's, the result carries no autograd graph: forward() computes the gradient."""
        plan = ops.FacePlan(imgs.shape, recs.shape, bboxes, keep=None)
        if plan.F == 0:
            return None
        return ops.face_crops(imgs, recs, plan)
