"""Shared by tests/test_host_b1_conv.py and tests/test_gpu_b1_conv.py: the conv shapes of the binary tensor-core
kernel (DESIGN.md §4x) and the launches a loaded 1-bit model makes on it."""

# (N, Cin, Cout, input side, stride): every qualifying layer shape of ImageNet ResNet-18/34 (224²), CIFAR ResNet-18
# (32²) and VGG-Small at small N, odd sizes, and ImageNet ResNet-18's layer2/3/4 shapes at N = 256
B1_SHAPES = [
    (2, 128, 128, 28, 1), (2, 128, 256, 28, 2), (2, 256, 256, 14, 1), (2, 256, 512, 14, 2), (2, 512, 512, 7, 1),
    (3, 128, 128, 16, 1), (3, 128, 256, 16, 2), (3, 256, 256, 8, 1), (3, 256, 512, 8, 2), (3, 512, 512, 4, 1),
    (2, 128, 128, 32, 1), (2, 128, 256, 16, 1), (2, 256, 256, 16, 1), (2, 256, 512, 8, 1), (2, 512, 512, 8, 1),
    (1, 128, 64, 9, 1), (2, 256, 128, 5, 2), (1, 512, 64, 3, 2), (3, 128, 128, 1, 1), (1, 256, 64, 11, 2),
    (256, 128, 128, 28, 1), (256, 128, 256, 28, 2), (256, 256, 256, 14, 1), (256, 256, 512, 14, 2),
    (256, 512, 512, 7, 1),
]

# binary tensor-core launches of one forward of a loaded 1-bit model: ResNet-18's layer2 (but layer2.0.conv1, 64
# input channels), layer3 and layer4; ResNet-34's likewise; VGG-Small's conv2 / conv4 as eval units and conv1 / conv3
# / conv5 as pooled int16 forwards; none in ResNet-20 (16-64 channels)
B1_MODEL_LAUNCHES = {
    "resnet18": {"binconv_fwd_b1_eval": 11, "binconv_fwd_b1_i16": 0},
    "resnet34": {"binconv_fwd_b1_eval": 25, "binconv_fwd_b1_i16": 0},
    "vgg_small": {"binconv_fwd_b1_eval": 2, "binconv_fwd_b1_i16": 3},
    "resnet20": {"binconv_fwd_b1_eval": 0, "binconv_fwd_b1_i16": 0},
}


def b1_shape_ok(cin, cout, kernel, stride, padding):
    """BDBNN_TC_B1's geometry: 3x3, pad 1, stride 1 or 2, Cin 128/256/512, Cout % 64 == 0."""
    return kernel == 3 and padding == 1 and stride in (1, 2) and cin in (128, 256, 512) and cout % 64 == 0
