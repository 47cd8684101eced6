"""Workload models (the reference's workloads live in external images:
tf_cnn_benchmarks ResNet-101, examples/v2beta1/tensorflow-benchmarks/
tensorflow-benchmarks.yaml:38-42; Horovod MNIST, examples/v2beta1/horovod/
tensorflow_mnist.py:38-73).  Model compute stays in PyTorch/cuDNN; the
hand-written sm_90a surface is the collective + optimizer path."""
from .resnet import resnet18, resnet50, resnet101, resnet152, ResNet  # noqa: F401
from .mnist import MnistConvNet  # noqa: F401
from .classic import trivial, lenet, alexnet, vgg11, vgg16, vgg19  # noqa: F401

MODEL_REGISTRY = {
    "resnet18": resnet18, "resnet50": resnet50, "resnet101": resnet101, "resnet152": resnet152,
    "mnist": MnistConvNet,
    "trivial": trivial, "lenet": lenet, "alexnet": alexnet, "vgg11": vgg11, "vgg16": vgg16, "vgg19": vgg19,
}


# tf_cnn_benchmarks model names (its --model flag) that are not written in-tree map onto torchvision definitions: cuDNN /
# ATen compute without the fused BN kernels, same trainer and collectives. Any other torchvision constructor name works too.
_TORCHVISION_ALIASES = {
    "inception3": ("inception_v3", {"aux_logits": False, "init_weights": False}),
    "googlenet": ("googlenet", {"aux_logits": False, "init_weights": False}),
    "mobilenet": ("mobilenet_v2", {}),
    "densenet121": ("densenet121", {}),
    "resnet34": ("resnet34", {}),
    "resnet50_v1.5": None,     # the in-tree ResNet already strides in the 3x3 (v1.5)
    "resnet101_v1.5": None,
    "resnet152_v1.5": None,
}


def model_names():
    return sorted(set(MODEL_REGISTRY) | set(_TORCHVISION_ALIASES))


def build_model(name: str, **kw):
    if name in MODEL_REGISTRY:
        return MODEL_REGISTRY[name](**kw)
    if name in _TORCHVISION_ALIASES and _TORCHVISION_ALIASES[name] is None:
        return MODEL_REGISTRY[name.split("_v1.5")[0]](**kw)
    try:
        import torchvision
    except ImportError:
        torchvision = None
    if torchvision is not None:
        ctor, defaults = _TORCHVISION_ALIASES.get(name, (name, {}))
        fn = getattr(torchvision.models, ctor, None)
        if callable(fn) and not isinstance(fn, type):
            return fn(weights=None, **{**defaults, **kw})
    raise KeyError(f"unknown model {name!r}; have {model_names()} (and torchvision.models constructors)")
