"""Zero-argument CIFAR builders looked up at train.py:50-52,257,285: `cifar_models.__dict__[arch]()`."""
from bdbnn_b200.resnet import resnet18_cifar as resnet18  # noqa: F401
from bdbnn_b200.resnet import resnet20  # noqa: F401
from bdbnn_b200.vgg import vgg_small  # noqa: F401
