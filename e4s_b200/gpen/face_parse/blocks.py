"""Building blocks of GPEN's ParseNet: mirror of src/pretrained/gpen/face_parse/blocks.py (NormLayer, ReluLayer, ConvLayer,
ResidualBlock).

The module trees, constructor arguments and parameter / buffer names are the reference's, so a ``ParseNet-latest.pth`` loads
with strict=True.  The blocks have no forward of their own: ``ParseNet.forward`` runs the whole network on the e4s_b200
kernels (parse_model.py).
"""
import numpy as np
from torch import nn
from torch.nn import functional as F


class NormLayer(nn.Module):
    """Normalization layer (run by ParseNet.forward; 'bn' is folded into the convolution before it)."""

    def __init__(self, channels, normalize_shape=None, norm_type='bn', ref_channels=None):
        super(NormLayer, self).__init__()
        norm_type = norm_type.lower()
        self.norm_type = norm_type
        if norm_type == 'bn':
            self.norm = nn.BatchNorm2d(channels, affine=True)
        elif norm_type == 'in':
            self.norm = nn.InstanceNorm2d(channels, affine=False)
        elif norm_type == 'gn':
            self.norm = nn.GroupNorm(32, channels, affine=True)
        elif norm_type == 'pixel':
            self.norm = lambda x: F.normalize(x, p=2, dim=1)
        elif norm_type == 'layer':
            self.norm = nn.LayerNorm(normalize_shape)
        elif norm_type == 'none':
            self.norm = lambda x: x * 1.0
        else:
            assert 1 == 0, 'Norm type {} not support.'.format(norm_type)


class ReluLayer(nn.Module):
    """Activation layer (run by ParseNet.forward; 'leakyrelu' is slope 0.2 in the convolution's epilogue)."""

    def __init__(self, channels, relu_type='relu'):
        super(ReluLayer, self).__init__()
        relu_type = relu_type.lower()
        self.relu_type = relu_type
        if relu_type == 'relu':
            self.func = nn.ReLU(True)
        elif relu_type == 'leakyrelu':
            self.func = nn.LeakyReLU(0.2, inplace=True)
        elif relu_type == 'prelu':
            self.func = nn.PReLU(channels)
        elif relu_type == 'selu':
            self.func = nn.SELU(True)
        elif relu_type == 'none':
            self.func = lambda x: x * 1.0
        else:
            assert 1 == 0, 'Relu type {} not support.'.format(relu_type)


class ConvLayer(nn.Module):
    """Scale ('up': nearest 2x first; 'down': stride 2), reflection pad, convolution, norm, activation (run by
    ParseNet.forward)."""

    def __init__(self, in_channels, out_channels, kernel_size=3, scale='none', norm_type='none', relu_type='none', use_pad=True,
                 bias=True):
        super(ConvLayer, self).__init__()
        self.use_pad = use_pad
        self.norm_type = norm_type
        if norm_type in ['bn']:
            bias = False

        stride = 2 if scale == 'down' else 1
        self.scale = scale

        self.scale_func = lambda x: x
        if scale == 'up':
            self.scale_func = lambda x: nn.functional.interpolate(x, scale_factor=2, mode='nearest')

        self.reflection_pad = nn.ReflectionPad2d(int(np.ceil((kernel_size - 1.) / 2)))
        self.conv2d = nn.Conv2d(in_channels, out_channels, kernel_size, stride, bias=bias)

        self.relu = ReluLayer(out_channels, relu_type)
        self.norm = NormLayer(out_channels, norm_type=norm_type)


class ResidualBlock(nn.Module):
    """identity + conv2(conv1(x)), the identity a ConvLayer when the block scales or changes the channel count (run by
    ParseNet.forward)."""

    def __init__(self, c_in, c_out, relu_type='prelu', norm_type='bn', scale='none'):
        super(ResidualBlock, self).__init__()
        self.scale = scale

        if scale == 'none' and c_in == c_out:
            self.shortcut_func = lambda x: x
        else:
            self.shortcut_func = ConvLayer(c_in, c_out, 3, scale)

        scale_config_dict = {'down': ['none', 'down'], 'up': ['up', 'none'], 'none': ['none', 'none']}
        scale_conf = scale_config_dict[scale]

        self.conv1 = ConvLayer(c_in, c_out, 3, scale_conf[0], norm_type=norm_type, relu_type=relu_type)
        self.conv2 = ConvLayer(c_out, c_out, 3, scale_conf[1], norm_type=norm_type, relu_type='none')
