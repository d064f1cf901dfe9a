"""MinkUNet (model/mink_unet.py, model/resnet_base.py of the reference) on the sparse convolution of ``sparse.py``.

The layer structure, forward, ``cat`` order, BatchNorm momentum and initialisation follow the reference, and
``state_dict()`` has the reference module's keys and shapes, so ``model.load_state_dict(torch.load(ckpt))`` loads a
reference checkpoint.  Weights trained with MinkowskiEngine itself are only right if its kernel-offset order is the
one ``sparse.py`` documents; that has not been checked against MinkowskiEngine.  Checkpoints trained with this module
are self-consistent.  The output ``.F`` at tensor stride 1 is in input row order."""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from .sparse import BatchNorm, Convolution, ConvolutionTranspose, ReLU, SparseTensor, cat


class BasicBlock(nn.Module):
    """MinkowskiEngine.modules.resnet_block.BasicBlock: two 3x3x3 convolutions, a residual and a ReLU."""
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, dilation=1, downsample=None, bn_momentum=0.1, dimension=-1):
        super().__init__()
        self.conv1 = Convolution(inplanes, planes, kernel_size=3, stride=stride, dilation=dilation, dimension=dimension)
        self.norm1 = BatchNorm(planes, momentum=bn_momentum)
        self.conv2 = Convolution(planes, planes, kernel_size=3, stride=1, dilation=dilation, dimension=dimension)
        self.norm2 = BatchNorm(planes, momentum=bn_momentum)
        self.relu = ReLU(inplace=True)
        self.downsample = downsample

    def forward(self, x: SparseTensor) -> SparseTensor:
        residual = x
        out = self.relu(self.norm1(self.conv1(x)))
        out = self.norm2(self.conv2(out))
        if self.downsample is not None:
            residual = self.downsample(x)
        return self.relu(out + residual)


def _kaiming_normal_fan_out(kernel):
    """ME.utils.kaiming_normal_(kernel, mode="fan_out", nonlinearity="relu"): std sqrt(2 / (C_out * K))."""
    K = kernel.shape[0] if kernel.dim() == 3 else 1
    std = math.sqrt(2.0) / math.sqrt(kernel.shape[-1] * K)
    with torch.no_grad():
        kernel.normal_(0, std)


class MinkUNetBase(nn.Module):
    BLOCK = BasicBlock
    PLANES = None
    LAYERS = (2, 2, 2, 2, 2, 2, 2, 2)
    INIT_DIM = 32

    def __init__(self, in_channels, out_channels, D=3):
        super().__init__()
        if D != 3:
            raise NotImplementedError(f"D = {D}: only 3-D networks are supported")
        self.D = D
        self.network_initialization(in_channels, out_channels, D)
        self.weight_initialization()

    def network_initialization(self, in_channels, out_channels, D):
        P, B = self.PLANES, self.BLOCK
        self.inplanes = self.INIT_DIM
        self.conv0p1s1 = Convolution(in_channels, self.inplanes, kernel_size=5, dimension=D)
        self.bn0 = BatchNorm(self.inplanes)
        self.conv1p1s2 = Convolution(self.inplanes, self.inplanes, kernel_size=2, stride=2, dimension=D)
        self.bn1 = BatchNorm(self.inplanes)
        self.block1 = self._make_layer(B, P[0], self.LAYERS[0])
        self.conv2p2s2 = Convolution(self.inplanes, self.inplanes, kernel_size=2, stride=2, dimension=D)
        self.bn2 = BatchNorm(self.inplanes)
        self.block2 = self._make_layer(B, P[1], self.LAYERS[1])
        self.conv3p4s2 = Convolution(self.inplanes, self.inplanes, kernel_size=2, stride=2, dimension=D)
        self.bn3 = BatchNorm(self.inplanes)
        self.block3 = self._make_layer(B, P[2], self.LAYERS[2])
        self.conv4p8s2 = Convolution(self.inplanes, self.inplanes, kernel_size=2, stride=2, dimension=D)
        self.bn4 = BatchNorm(self.inplanes)
        self.block4 = self._make_layer(B, P[3], self.LAYERS[3])
        self.convtr4p16s2 = ConvolutionTranspose(self.inplanes, P[4], kernel_size=2, stride=2, dimension=D)
        self.bntr4 = BatchNorm(P[4])
        self.inplanes = P[4] + P[2] * B.expansion
        self.block5 = self._make_layer(B, P[4], self.LAYERS[4])
        self.convtr5p8s2 = ConvolutionTranspose(self.inplanes, P[5], kernel_size=2, stride=2, dimension=D)
        self.bntr5 = BatchNorm(P[5])
        self.inplanes = P[5] + P[1] * B.expansion
        self.block6 = self._make_layer(B, P[5], self.LAYERS[5])
        self.convtr6p4s2 = ConvolutionTranspose(self.inplanes, P[6], kernel_size=2, stride=2, dimension=D)
        self.bntr6 = BatchNorm(P[6])
        self.inplanes = P[6] + P[0] * B.expansion
        self.block7 = self._make_layer(B, P[6], self.LAYERS[6])
        self.convtr7p2s2 = ConvolutionTranspose(self.inplanes, P[7], kernel_size=2, stride=2, dimension=D)
        self.bntr7 = BatchNorm(P[7])
        self.inplanes = P[7] + self.INIT_DIM
        self.block8 = self._make_layer(B, P[7], self.LAYERS[7])
        self.final = Convolution(P[7], out_channels, kernel_size=1, dimension=D)
        self.relu = ReLU(inplace=True)

    def weight_initialization(self):
        # ResNetBase.weight_initialization: the transposed layers are not MinkowskiConvolution instances there either,
        # so they keep their default initialisation.
        for m in self.modules():
            if isinstance(m, Convolution):
                _kaiming_normal_fan_out(m.kernel)
            if isinstance(m, BatchNorm):
                nn.init.constant_(m.bn.weight, 1)
                nn.init.constant_(m.bn.bias, 0)

    def _make_layer(self, block, planes, blocks, stride=1, dilation=1, bn_momentum=0.1):
        downsample = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            downsample = nn.Sequential(
                Convolution(self.inplanes, planes * block.expansion, kernel_size=1, stride=stride, dimension=self.D),
                BatchNorm(planes * block.expansion))
        layers = [block(self.inplanes, planes, stride=stride, dilation=dilation, downsample=downsample,
                        dimension=self.D)]
        self.inplanes = planes * block.expansion
        for _ in range(1, blocks):
            layers.append(block(self.inplanes, planes, stride=1, dilation=dilation, dimension=self.D))
        return nn.Sequential(*layers)

    def forward(self, x: SparseTensor) -> SparseTensor:
        out_p1 = self.relu(self.bn0(self.conv0p1s1(x)))
        out = self.relu(self.bn1(self.conv1p1s2(out_p1)))
        out_b1p2 = self.block1(out)
        out = self.relu(self.bn2(self.conv2p2s2(out_b1p2)))
        out_b2p4 = self.block2(out)
        out = self.relu(self.bn3(self.conv3p4s2(out_b2p4)))
        out_b3p8 = self.block3(out)
        out = self.relu(self.bn4(self.conv4p8s2(out_b3p8)))
        out = self.block4(out)
        out = self.relu(self.bntr4(self.convtr4p16s2(out)))
        out = self.block5(cat(out, out_b3p8))
        out = self.relu(self.bntr5(self.convtr5p8s2(out)))
        out = self.block6(cat(out, out_b2p4))
        out = self.relu(self.bntr6(self.convtr6p4s2(out)))
        out = self.block7(cat(out, out_b1p2))
        out = self.relu(self.bntr7(self.convtr7p2s2(out)))
        out = self.block8(cat(out, out_p1))
        return self.final(out)


_ARCHS = {
    "MinkUNet14A": ((1,) * 8, (32, 64, 128, 256, 128, 128, 96, 96)),
    "MinkUNet14B": ((1,) * 8, (32, 64, 128, 256, 128, 128, 128, 128)),
    "MinkUNet14C": ((1,) * 8, (32, 64, 128, 256, 192, 192, 128, 128)),
    "MinkUNet14D": ((1,) * 8, (32, 64, 128, 256, 384, 384, 384, 384)),
    "MinkUNet18A": ((2,) * 8, (32, 64, 128, 256, 128, 128, 96, 96)),
    "MinkUNet18B": ((2,) * 8, (32, 64, 128, 256, 128, 128, 128, 128)),
    "MinkUNet18D": ((2,) * 8, (32, 64, 128, 256, 384, 384, 384, 384)),
    "MinkUNet34A": ((2, 3, 4, 6, 2, 2, 2, 2), (32, 64, 128, 256, 256, 128, 64, 64)),
    "MinkUNet34B": ((2, 3, 4, 6, 2, 2, 2, 2), (32, 64, 128, 256, 256, 128, 64, 32)),
    "MinkUNet34C": ((2, 3, 4, 6, 2, 2, 2, 2), (32, 64, 128, 256, 256, 128, 96, 96)),
}
ARCHS = tuple(_ARCHS)


def mink_unet(in_channels=3, out_channels=20, D=3, arch="MinkUNet18A") -> MinkUNetBase:
    """The reference's factory: every arch name it accepts (all BasicBlock)."""
    if arch not in _ARCHS:
        raise ValueError(f"architecture {arch!r} not supported; one of {', '.join(ARCHS)}")
    layers, planes = _ARCHS[arch]
    cls = type(arch, (MinkUNetBase,), {"LAYERS": layers, "PLANES": planes})
    return cls(in_channels, out_channels, D)
