"""ResNet (v1.5: stride on the 3x3 conv of the bottleneck), the model behind the
reference's headline synthetic benchmark.

A block's output feeds two consumers in the next block: conv1 and the skip path (the identity residual or the
downsample).  Inside ResNet.forward the blocks pass a ``(main, skip)`` pair, the last batch norm of a block returning
its output and an alias of it, so the two gradients reach that batch norm's backward separately and its kernel sums
them as it reads them (ops/bn_act.py).  The stem's batch norm does the same for the max-pooled output that feeds
layer1, and runs the ReLU and the max pool in its own kernels.  A block called on one tensor uses it for both and
returns one tensor."""
import torch
import torch.nn as nn

from ..ops.bn_act import BatchNormAct2d
from ..ops.stem_conv import StemConv2d


def _conv3x3(i, o, stride=1):
    return nn.Conv2d(i, o, 3, stride, 1, bias=False)


def _conv1x1(i, o, stride=1):
    return nn.Conv2d(i, o, 1, stride, bias=False)


class BasicBlock(nn.Module):
    expansion = 1

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = _conv3x3(inplanes, planes, stride)
        self.bn1 = BatchNormAct2d(planes, act="relu")
        self.conv2 = _conv3x3(planes, planes)
        self.bn2 = BatchNormAct2d(planes, act="relu")
        self.downsample = downsample

    def forward(self, x):
        main, skip = x if isinstance(x, tuple) else (x, x)
        idt = skip if self.downsample is None else self.downsample(skip)
        out = self.bn1(self.conv1(main))
        return self.bn2(self.conv2(out), idt, pair=isinstance(x, tuple))


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super().__init__()
        self.conv1 = _conv1x1(inplanes, planes)
        self.bn1 = BatchNormAct2d(planes, act="relu")
        self.conv2 = _conv3x3(planes, planes, stride)
        self.bn2 = BatchNormAct2d(planes, act="relu")
        self.conv3 = _conv1x1(planes, planes * 4)
        self.bn3 = BatchNormAct2d(planes * 4, act="relu")
        self.downsample = downsample

    def forward(self, x):
        main, skip = x if isinstance(x, tuple) else (x, x)
        idt = skip if self.downsample is None else self.downsample(skip)
        out = self.bn1(self.conv1(main))
        out = self.bn2(self.conv2(out))
        return self.bn3(self.conv3(out), idt, pair=isinstance(x, tuple))


class ResNet(nn.Module):
    def __init__(self, block, layers, num_classes=1000, zero_init_residual=False):
        super().__init__()
        self.inplanes = 64
        self.conv1 = StemConv2d(3, 64, 7, 2, 3, bias=False)
        self.bn1 = BatchNormAct2d(64, act="relu")
        self.maxpool = nn.MaxPool2d(3, 2, 1)
        self.layer1 = self._make_layer(block, 64, layers[0])
        self.layer2 = self._make_layer(block, 128, layers[1], 2)
        self.layer3 = self._make_layer(block, 256, layers[2], 2)
        self.layer4 = self._make_layer(block, 512, layers[3], 2)
        self.avgpool = nn.AdaptiveAvgPool2d((1, 1))
        self.fc = nn.Linear(512 * block.expansion, num_classes)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)
        if zero_init_residual:
            for m in self.modules():
                if isinstance(m, Bottleneck):
                    nn.init.zeros_(m.bn3.weight)
                elif isinstance(m, BasicBlock):
                    nn.init.zeros_(m.bn2.weight)

    def _make_layer(self, block, planes, blocks, stride=1):
        down = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            down = nn.Sequential(_conv1x1(self.inplanes, planes * block.expansion, stride),
                                 BatchNormAct2d(planes * block.expansion))
        layers = [block(self.inplanes, planes, stride, down)]
        self.inplanes = planes * block.expansion
        layers += [block(self.inplanes, planes) for _ in range(1, blocks)]
        return nn.Sequential(*layers)

    def forward(self, x):
        x = self.bn1(self.conv1(x), pool=self.maxpool, pair=True)   # the stem's batch norm, ReLU and max pool
        x, _ = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        return self.fc(torch.flatten(self.avgpool(x), 1))


def resnet18(**kw):
    return ResNet(BasicBlock, [2, 2, 2, 2], **kw)


def resnet34(**kw):
    return ResNet(BasicBlock, [3, 4, 6, 3], **kw)


def resnet50(**kw):
    return ResNet(Bottleneck, [3, 4, 6, 3], **kw)


def resnet101(**kw):
    return ResNet(Bottleneck, [3, 4, 23, 3], **kw)


def resnet152(**kw):
    return ResNet(Bottleneck, [3, 8, 36, 3], **kw)
