"""Table-driven mirror of the reference's sparse ResNets (``models/resnet_base.py:31-160``: ResNet14/18/34 on BasicBlock,
ResNet50/101 on Bottleneck), in the way ``minkunet.py`` mirrors the U-Net: the same attribute names (-> the same
state-dict keys: ``conv1.kernel``, ``bn1.bn.weight``, ``layer1.0.downsample.0.kernel``, ``conv5.kernel``,
``final.linear.weight``), the same construction order (-> the same seeded initialisation) and the same forward.

The network: a 5^3 stride-2 stem, 2^3 stride-2 average pooling, four stages of stride 2 (tensor stride 64), a 3^3 stride-3
convolution (tensor stride 192), global max pooling per batch index and a linear head.  ``forward`` returns the dense
``[B, out_channels]`` logits.  ``ME`` is the namespace providing the MinkowskiEngine surface (``minkunet.default_me()``
by default; tests pass the CPU oracle)."""
import torch.nn as nn

from .minkunet import default_me

# name -> (block, blocks per stage); resnet_base.py:141-160
ARCHS = {
    'ResNet14': ('basic', (1, 1, 1, 1)),
    'ResNet18': ('basic', (2, 2, 2, 2)),
    'ResNet34': ('basic', (3, 4, 6, 3)),
    'ResNet50': ('bottleneck', (3, 4, 6, 3)),
    'ResNet101': ('bottleneck', (3, 4, 23, 3)),
}
INIT_DIM = 64
PLANES = (64, 128, 256, 512)


class ResNet(nn.Module):
    def __init__(self, arch, in_channels, out_channels, D=3, ME=None):
        super().__init__()
        if arch not in ARCHS:
            raise ValueError(f"unknown ResNet {arch!r}; one of {sorted(ARCHS)}")
        ME = ME or default_me()
        block_kind, layers = ARCHS[arch]
        block = ME.BasicBlock if block_kind == 'basic' else ME.Bottleneck
        self.arch, self.D = arch, D
        width = INIT_DIM

        def stage(planes, n_blocks, stride):
            nonlocal width
            down = None
            if stride != 1 or width != planes * block.expansion:
                down = nn.Sequential(ME.MinkowskiConvolution(width, planes * block.expansion, kernel_size=1, stride=stride,
                                                             dimension=D),
                                     ME.MinkowskiBatchNorm(planes * block.expansion))
            blocks = [block(width, planes, stride=stride, dilation=1, downsample=down, dimension=D)]
            width = planes * block.expansion
            blocks += [block(width, planes, stride=1, dilation=1, dimension=D) for _ in range(1, n_blocks)]
            return nn.Sequential(*blocks)

        self.conv1 = ME.MinkowskiConvolution(in_channels, width, kernel_size=5, stride=2, dimension=D)
        self.bn1 = ME.MinkowskiBatchNorm(width)
        self.relu = ME.MinkowskiReLU(inplace=True)
        self.pool = ME.MinkowskiAvgPooling(kernel_size=2, stride=2, dimension=D)
        for i, (planes, n_blocks) in enumerate(zip(PLANES, layers)):
            setattr(self, f'layer{i + 1}', stage(planes, n_blocks, 2))
        self.conv5 = ME.MinkowskiConvolution(width, width, kernel_size=3, stride=3, dimension=D)
        self.bn5 = ME.MinkowskiBatchNorm(width)
        self.glob_avg = ME.MinkowskiGlobalMaxPooling(dimension=D)     # the reference's name for its global max pooling
        self.final = ME.MinkowskiLinear(width, out_channels, bias=True)

        # resnet_base.py:73-80
        for m in self.modules():
            if isinstance(m, ME.MinkowskiConvolution):
                ME.kaiming_normal_(m.kernel, mode='fan_out', nonlinearity='relu')
            if isinstance(m, ME.MinkowskiBatchNorm):
                nn.init.constant_(m.bn.weight, 1)
                nn.init.constant_(m.bn.bias, 0)

    def forward(self, x):
        x = self.pool(self.relu(self.bn1(self.conv1(x))))
        for i in range(1, 5):
            x = getattr(self, f'layer{i}')(x)
        x = self.relu(self.bn5(self.conv5(x)))
        return self.final(self.glob_avg(x))


def resnet(arch='ResNet18', in_channels=3, out_channels=20, D=3, ME=None):
    return ResNet(arch, in_channels, out_channels, D, ME=ME)
