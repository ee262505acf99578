"""Lower-case, callable model builders looked up by name at train.py:53-56,253,283:
`imagenet_models.__dict__[args.arch](pretrained)`."""
from bdbnn_b200.resnet import resnet18, resnet18_step1, resnet34, resnet34_step1  # noqa: F401
from . import resnet_bi_imagenet_set_2, resnet_bi_imagenet_set_2_2  # noqa: F401
