"""Parameter container mirroring audio_zen/model/module/sequence_model.py:26-125.

The ``nn.LSTM`` / ``nn.Linear`` members exist only to own the parameters with PyTorch's names,
shapes and default initialisation, so ``state_dict`` keys (``sequence_model.weight_ih_l0`` ...,
``fc_output_layer.weight``), checkpoints, ``torch.optim.Adam`` and DDP behave exactly as with the
reference.  Their ``forward`` is never called: the arithmetic runs in libfsn_b200."""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn

from ... import _lib

LSTM_PARAMS = ("weight_ih", "weight_hh", "bias_ih", "bias_hh")  # in the field order of fsn_lstm_layer / fsn_lstm_grads


class SequenceModel(nn.Module):
    def __init__(self, input_size, output_size, hidden_size, num_layers, bidirectional,
                 sequence_model="GRU", output_activate_function="Tanh"):
        super().__init__()
        if sequence_model == "LSTM":
            self.sequence_model = nn.LSTM(input_size=input_size, hidden_size=hidden_size, num_layers=num_layers,
                                          batch_first=True, bidirectional=bidirectional)
        elif sequence_model == "GRU":  # sequence_model.py:59-66 (weights [3H,K], gate order r,z,n)
            self.sequence_model = nn.GRU(input_size=input_size, hidden_size=hidden_size, num_layers=num_layers,
                                         batch_first=True, bidirectional=bidirectional)
        else:
            raise NotImplementedError(f"Not implemented {sequence_model}")  # sequence_model.py:67-68
        self.cell = sequence_model
        if bidirectional or not 1 <= num_layers <= 8:
            raise NotImplementedError("libfsn_b200 builds uni-directional LSTM / GRU stacks of 1..8 layers")
        if int(output_size):  # sequence_model.py:82-84 (no Linear layer when output_size == 0)
            self.fc_output_layer = nn.Linear(hidden_size, output_size)
        self.num_layers = num_layers
        if output_activate_function:
            if output_activate_function not in ("Tanh", "ReLU", "ReLU6"):
                raise NotImplementedError(f"Not implemented activation function {output_activate_function}")
        self.output_activate_function = output_activate_function
        self.output_size = output_size
        self.input_size, self.hidden_size = input_size, hidden_size

    @staticmethod
    def _check(p, name):
        if not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous():
            raise RuntimeError(f"fullsubnet_b200: parameter {name} must be a contiguous fp32 CUDA tensor "
                               f"(got {p.device}, {p.dtype}); call model.cuda() first - there is no CPU path.")
        return p.data_ptr()

    def layer_struct(self, l: int = 0) -> "_lib.LstmLayer":
        """Raw device pointers of LSTM layer ``l`` (fsn_lstm_layer)."""
        lstm = self.sequence_model
        return _lib.LstmLayer(*(self._check(getattr(lstm, f"{n}_l{l}"), f"{n}_l{l}") for n in LSTM_PARAMS))

    @staticmethod
    def grads_struct(grads: dict, prefix: str, l: int) -> "_lib.LstmGrads":
        """Pointers of the gradients of LSTM layer ``l`` (fsn_lstm_grads), from named gradient tensors; ``prefix`` is
        the SequenceModel's name in the model followed by a dot."""
        return _lib.LstmGrads(*(grads[f"{prefix}sequence_model.{n}_l{l}"].data_ptr() for n in LSTM_PARAMS))

    @staticmethod
    def seq_grads_struct(grads: dict, prefix: str) -> "_lib.SeqGrads":
        """Pointers of the gradients of a 2-layer stack with its Linear (fsn_seq_grads), from named gradient tensors;
        ``prefix`` is the SequenceModel's name in the model followed by a dot."""
        g = _lib.SeqGrads()
        for l in range(2):
            lg = SequenceModel.grads_struct(grads, prefix, l)
            for field in ("w_ih", "w_hh", "b_ih", "b_hh"):
                getattr(g, field)[l] = getattr(lg, field)
        g.fc_w = grads[f"{prefix}fc_output_layer.weight"].data_ptr()
        g.fc_b = grads[f"{prefix}fc_output_layer.bias"].data_ptr()
        return g

    def fc_ptrs(self):
        return (self._check(self.fc_output_layer.weight, "fc_output_layer.weight"),
                self._check(self.fc_output_layer.bias, "fc_output_layer.bias"))

    def weight_struct(self) -> "_lib.SeqWeights":
        """Raw device pointers into the parameter storage (fsn_seq_weights)."""
        assert self.num_layers == 2 and hasattr(self, "fc_output_layer")
        w = _lib.SeqWeights()
        for l in range(2):
            layer = self.layer_struct(l)
            for field in ("w_ih", "w_hh", "b_ih", "b_hh"):
                getattr(w, field)[l] = getattr(layer, field)
        w.fc_w, w.fc_b = self.fc_ptrs()
        return w

    def version_key(self):
        return tuple((p.data_ptr(), p._version) for p in self.parameters())

    def forward(self, x):  # pragma: no cover - never on the product path
        raise RuntimeError("SequenceModel is a parameter container in fullsubnet_b200; call Model.forward")
