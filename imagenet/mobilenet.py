"""MobileNet-v1 encoder definition (module surface only).

Mirrors the public surface of the reference's ``imagenet/mobilenet.py``
(reference imagenet/mobilenet.py:12-62): a ``MobileNet(relu6=True)`` module whose
``.model`` is an ``nn.Sequential`` of one dense 3x3/s2 stem block followed by
13 depthwise-separable blocks and an ``AvgPool2d(7)``, plus an ``fc`` head.
The depth networks in ``models.py`` only consume ``model[0..13]``
(reference models.py:674-675).

State-dict keys are identical to the reference (``model.<i>.<0|1|3|4>.*``,
``fc.*``) so ImageNet checkpoints written by the reference load unchanged.
Nothing here runs on the hot path: on CUDA the blocks are *read* by
``fastdepth_b200.plan`` (conv weight + BN statistics) and executed by the
sm_90a kernels.

Extension over the reference: ``widths`` lets callers build NetAdapt-pruned
encoders (SURVEY.md section 8a-a10); the default reproduces the stock widths.
"""
import torch.nn as nn

# (out_channels, stride) of blocks 0..13; block 0 is the dense stem.
# Strides follow reference imagenet/mobilenet.py:41-54.
STOCK_WIDTHS = (32, 64, 128, 128, 256, 256, 512, 512, 512, 512, 512, 512, 1024, 1024)
STRIDES = (2, 1, 2, 1, 2, 1, 2, 1, 1, 1, 1, 1, 2, 1)


def _act(relu6):
    return nn.ReLU6(inplace=True) if relu6 else nn.ReLU(inplace=True)


def stem_block(c_in, c_out, stride, relu6=True):
    """Dense 3x3 conv + BN + activation (reference imagenet/mobilenet.py:22-27)."""
    return nn.Sequential(
        nn.Conv2d(c_in, c_out, kernel_size=3, stride=stride, padding=1, bias=False),
        nn.BatchNorm2d(c_out),
        _act(relu6))


def separable_block(c_in, c_out, stride, relu6=True):
    """dw3x3(stride)+BN+act -> pw1x1+BN+act (reference imagenet/mobilenet.py:29-38)."""
    return nn.Sequential(
        nn.Conv2d(c_in, c_in, kernel_size=3, stride=stride, padding=1, groups=c_in, bias=False),
        nn.BatchNorm2d(c_in),
        _act(relu6),
        nn.Conv2d(c_in, c_out, kernel_size=1, stride=1, padding=0, bias=False),
        nn.BatchNorm2d(c_out),
        _act(relu6))


class MobileNet(nn.Module):
    def __init__(self, relu6=True, widths=None, in_channels=3, num_classes=1000):
        super().__init__()
        widths = tuple(widths) if widths is not None else STOCK_WIDTHS
        if len(widths) != len(STRIDES):
            raise ValueError("need %d encoder widths, got %d" % (len(STRIDES), len(widths)))
        blocks = [stem_block(in_channels, widths[0], STRIDES[0], relu6)]
        for i in range(1, len(widths)):
            blocks.append(separable_block(widths[i - 1], widths[i], STRIDES[i], relu6))
        blocks.append(nn.AvgPool2d(7))
        self.model = nn.Sequential(*blocks)
        self.fc = nn.Linear(widths[-1], num_classes)

    def forward(self, x):
        x = self.model(x)
        return self.fc(x.flatten(1))
