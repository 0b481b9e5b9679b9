"""ResNet-18 trunk of the BiSeNet face parser: mirror of src/pretrained/face_parsing/resnet.py.

The module tree and parameter names are the reference's, so ``79999_iter.pth`` loads.  Unlike the reference, constructing
``Resnet18()`` downloads nothing: the reference fetches ImageNet weights at construction (resnet.py:83), which loading the
parser's checkpoint overwrites anyway.  These modules hold parameters only; ``BiSeNet.forward`` (model.py) runs them on the
library's kernels.
"""
from torch import nn


def conv3x3(in_planes, out_planes, stride=1):
    """3x3 convolution, padding 1, no bias."""
    return nn.Conv2d(in_planes, out_planes, kernel_size=3, stride=stride, padding=1, bias=False)


class BasicBlock(nn.Module):
    def __init__(self, in_chan, out_chan, stride=1):
        super().__init__()
        self.conv1 = conv3x3(in_chan, out_chan, stride)
        self.bn1 = nn.BatchNorm2d(out_chan)
        self.conv2 = conv3x3(out_chan, out_chan)
        self.bn2 = nn.BatchNorm2d(out_chan)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = None
        if in_chan != out_chan or stride != 1:
            self.downsample = nn.Sequential(nn.Conv2d(in_chan, out_chan, kernel_size=1, stride=stride, bias=False),
                                            nn.BatchNorm2d(out_chan))


def create_layer_basic(in_chan, out_chan, bnum, stride=1):
    return nn.Sequential(BasicBlock(in_chan, out_chan, stride=stride),
                         *[BasicBlock(out_chan, out_chan, stride=1) for _ in range(bnum - 1)])


class Resnet18(nn.Module):
    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 64, kernel_size=7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        self.layer1 = create_layer_basic(64, 64, bnum=2, stride=1)
        self.layer2 = create_layer_basic(64, 128, bnum=2, stride=2)
        self.layer3 = create_layer_basic(128, 256, bnum=2, stride=2)
        self.layer4 = create_layer_basic(256, 512, bnum=2, stride=2)
