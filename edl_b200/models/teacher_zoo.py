"""Named teacher models for ``python -m paddle_edl.distill.teacher_server --model NAME``.
``build(name) -> (module, feed_names, fetch_names, feed_shapes)``; the fetch name of the image
teachers is ``score`` (softmax probabilities), matching the reference's serving model
(example/distill/resnet/train_with_fleet.py:446).  The sequence teachers (``ernie_base``, ``minilm_l12_h384``,
``ernie_tiny``) take the reference's four ERNIE feeds as its ``ernie_reader`` batches them -- ``input_ids``,
``position_ids``, ``segment_ids`` int64 [L, 1] and ``input_mask`` float [L, 1] per sample -- and fetch ``logits``, fp32
[B, num_labels]."""
import torch
import torch.nn as nn

ERNIE_MAX_SEQ_LEN = 256    # the reference's max_seq_len for the ERNIE teacher


class _Probs(nn.Module):
    def __init__(self, net, channels_last=True):
        super().__init__()
        self.net, self.channels_last = net, channels_last

    @torch.no_grad()
    def forward(self, x):
        if x.dim() == 4 and self.channels_last:
            x = x.contiguous(memory_format=torch.channels_last)
        return torch.softmax(self.net(x).float(), -1)


def build(name):
    name = name.lower()
    if name in ("resnext101_32x16d", "resnext101_32x16d_wsl"):
        from .resnext import ResNeXt101_32x16d
        return _Probs(ResNeXt101_32x16d()), ["image"], ["score"], {"image": [3, 224, 224]}
    if name == "resnext50_32x4d":
        from .resnext import ResNeXt50_32x4d
        return _Probs(ResNeXt50_32x4d()), ["image"], ["score"], {"image": [3, 224, 224]}
    if name == "resnext_tiny":
        from .resnext import ResNeXt_tiny
        return _Probs(ResNeXt_tiny()), ["image"], ["score"], {"image": [3, 64, 64]}
    if name == "mnist_cnn":
        from .small import MnistTeacher
        return _Probs(MnistTeacher(), channels_last=False), ["img"], ["fc_0.tmp_2"], {"img": [1, 28, 28]}
    if name in ("ernie_base", "minilm_l12_h384", "ernie_tiny"):
        from . import ernie
        net = {"ernie_base": ernie.ernie_base, "minilm_l12_h384": ernie.minilm_l12_h384,
               "ernie_tiny": ernie.ernie_tiny}[name]()
        feeds = ["input_ids", "position_ids", "segment_ids", "input_mask"]
        return net, feeds, ["logits"], {f: [ERNIE_MAX_SEQ_LEN, 1] for f in feeds}
    raise ValueError("unknown teacher model %r" % name)
