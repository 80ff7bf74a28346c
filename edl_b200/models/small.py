"""Small workloads of the reference's examples: fit_a_line regression, the MNIST distill student and
teacher CNNs, the BOW / CNN NLP distill students and the bidirectional LSTM student.

References: example/fit_a_line/fluid/fit_a_line.py:33-44 (``fc(13 -> 1)``);
example/distill/mnist_distill/train_with_fleet.py:134-145 (LeNet-ish student, served CNN teacher);
example/distill/nlp/model.py:84-135 (BOW / CNN students)."""
import torch
import torch.nn as nn
import torch.nn.functional as F


class FitALine(nn.Module):
    def __init__(self, in_features=13):
        super().__init__()
        self.fc = nn.Linear(in_features, 1)

    def forward(self, x):
        return self.fc(x)


class MnistStudent(nn.Module):
    """conv-pool x2 + fc, the small student of the MNIST distill example."""

    def __init__(self, num_classes=10):
        super().__init__()
        self.conv1 = nn.Conv2d(1, 20, 5)
        self.conv2 = nn.Conv2d(20, 50, 5)
        self.fc = nn.Linear(50 * 4 * 4, num_classes)

    def forward(self, x):
        x = F.max_pool2d(F.relu(self.conv1(x)), 2)
        x = F.max_pool2d(F.relu(self.conv2(x)), 2)
        return self.fc(x.flatten(1))


class MnistTeacher(nn.Module):
    """A wider CNN playing the served teacher (the reference downloads a pre-trained serving model)."""

    def __init__(self, num_classes=10):
        super().__init__()
        self.features = nn.Sequential(nn.Conv2d(1, 32, 3, padding=1), nn.ReLU(), nn.Conv2d(32, 64, 3, padding=1),
                                      nn.ReLU(), nn.MaxPool2d(2), nn.Conv2d(64, 128, 3, padding=1), nn.ReLU(),
                                      nn.MaxPool2d(2))
        self.fc = nn.Sequential(nn.Linear(128 * 7 * 7, 256), nn.ReLU(), nn.Linear(256, num_classes))

    def forward(self, x):
        return self.fc(self.features(x).flatten(1))


class BOW(nn.Module):
    """Bag-of-words sentiment student: embedding -> sum-pool -> tanh -> fc -> fc(2)."""

    def __init__(self, vocab_size=30000, emb_dim=128, hid_dim=128, num_labels=2, padding_idx=0):
        super().__init__()
        self.emb = nn.Embedding(vocab_size, emb_dim, padding_idx=padding_idx)
        self.fc1 = nn.Linear(emb_dim, hid_dim)
        self.fc2 = nn.Linear(hid_dim, num_labels)
        self.padding_idx = padding_idx

    def forward(self, ids):
        mask = (ids != self.padding_idx).unsqueeze(-1)
        h = torch.tanh((self.emb(ids) * mask).sum(1))
        return self.fc2(torch.tanh(self.fc1(h)))


class TextCNN(nn.Module):
    """1-D CNN sentiment student: embedding -> conv(k=3) -> max-over-time -> fc(2)."""

    def __init__(self, vocab_size=30000, emb_dim=128, num_filters=128, kernel=3, num_labels=2, padding_idx=0):
        super().__init__()
        self.emb = nn.Embedding(vocab_size, emb_dim, padding_idx=padding_idx)
        self.conv = nn.Conv1d(emb_dim, num_filters, kernel, padding=kernel // 2)
        self.fc = nn.Linear(num_filters, num_labels)

    def forward(self, ids):
        h = torch.tanh(self.conv(self.emb(ids).transpose(1, 2))).max(-1).values
        return self.fc(h)


class BiLSTM(nn.Module):
    """Bidirectional LSTM sentiment student: embedding -> ``ops.lstm`` -> [h_n forward | h_n reverse] -> tanh(fc1) -> fc2
    (the head of ``BOW``).  The LSTM parameters live in an ``nn.LSTM`` submodule used as their container, so state
    dicts of a torch-trained BiLSTM load unchanged; the recurrence itself runs on ``ops.lstm`` (csrc/lstm.cu on CUDA).
    A sample's length is its last non-pad position + 1, computed on the device; a pad inside a sentence is read as the
    zero embedding row, as ``BOW``'s masking does."""

    def __init__(self, vocab_size=30000, emb_dim=128, hidden=128, num_labels=2, padding_idx=0):
        super().__init__()
        self.emb = nn.Embedding(vocab_size, emb_dim, padding_idx=padding_idx)
        self.lstm = nn.LSTM(emb_dim, hidden, batch_first=True, bidirectional=True)
        self.fc1 = nn.Linear(2 * hidden, hidden)
        self.fc2 = nn.Linear(hidden, num_labels)
        self.padding_idx = padding_idx

    def lstm_params(self):
        return [getattr(self.lstm, n) for n in ("weight_ih_l0", "weight_hh_l0", "bias_ih_l0", "bias_hh_l0",
                                                "weight_ih_l0_reverse", "weight_hh_l0_reverse",
                                                "bias_ih_l0_reverse", "bias_hh_l0_reverse")]

    def lengths(self, ids):
        pos = torch.arange(1, ids.shape[1] + 1, device=ids.device)
        return ((ids != self.padding_idx) * pos).amax(1)

    def forward(self, ids):
        from .. import ops

        x = self.emb(ids)
        if x.is_cuda:
            x = x.to(torch.bfloat16)
        _, h_n = ops.lstm(x, self.lengths(ids), self.lstm_params())
        h = torch.cat([h_n[0], h_n[1]], -1).to(self.fc1.weight.dtype)
        return self.fc2(torch.tanh(self.fc1(h)))


def kl_distill_loss(student_logits, teacher_logits, temperature=1.0):
    """``KL_T`` of the NLP example (T=2 there): KL(softmax(t/T) || softmax(s/T)) * T^2, on the fused
    soft-CE kernel when the tensors are on the GPU."""
    from .. import ops

    return ops.soft_cross_entropy(student_logits, teacher_logits, target_kind="logits",
                                  student_temperature=temperature, teacher_temperature=temperature, kl=True,
                                  loss_scale=temperature * temperature)
