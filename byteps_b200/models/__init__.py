"""Benchmark model zoo: the architectures the reference's examples train
(/root/reference/example/pytorch/benchmark_byteps.py uses torchvision models;
its published numbers are ResNet-50, VGG-16 and BERT-large).  Random-init,
synthetic-data friendly, channels_last / bf16 ready."""
from .bert import BertConfig, BertForPreTraining, bert_base, bert_large, bert_tiny  # noqa: F401
from .gpt import GptConfig, GptLMHeadModel, gpt2_medium, gpt2_small, gpt_tiny  # noqa: F401
from .mnist import MnistNet  # noqa: F401
from .resnet import ResNet, resnet18, resnet34, resnet50, resnet101, resnet152  # noqa: F401
from .vgg import VGG, vgg16, vgg19  # noqa: F401


def get_model(name: str, **kw):
    table = {
        "resnet18": resnet18, "resnet34": resnet34, "resnet50": resnet50, "resnet101": resnet101,
        "resnet152": resnet152, "vgg16": vgg16, "vgg19": vgg19, "bert_base": bert_base, "bert_large": bert_large,
        "bert_tiny": bert_tiny, "gpt_tiny": gpt_tiny, "gpt2_small": gpt2_small, "gpt2_medium": gpt2_medium,
        "mnist": MnistNet,
    }
    if name not in table:
        raise ValueError("unknown model %r (have: %s)" % (name, ", ".join(sorted(table))))
    return table[name](**kw)
