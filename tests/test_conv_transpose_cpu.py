"""`QuantConvTranspose2d` on the CPU side (SURVEY 8 row f4): module surface / prepare() of all three schemes without a GPU.
The reference's own wbwtab / dorefa classes are not runnable under current PyTorch (they hand dilation / groups / bias to
nn.ConvTranspose2d positionally in the wrong order), which is why only the IAO one (IAO:510-636) has golden fixtures generated
from the reference (tests/golden/layer_iao_convT_*.npz) and the other two are pinned on the oracle's quantizers composed with
ATen."""
import copy

import pytest
import torch
import torch.nn as nn


def _net():
    return nn.Sequential(nn.Conv2d(3, 16, 3, padding=1), nn.ReLU(), nn.ConvTranspose2d(16, 8, 4, stride=2, padding=1), nn.ReLU(),
                         nn.Conv2d(8, 4, 1))


def test_prepare_swaps_conv_transpose_in_every_scheme():
    from micronet_b200 import dorefa, iao, wbwtab
    base = _net()
    keys = list(base.state_dict().keys())
    d = dorefa.prepare(copy.deepcopy(base), a_bits=4, w_bits=4)
    assert isinstance(d[2], dorefa.QuantConvTranspose2d) and isinstance(d[2], nn.ConvTranspose2d)
    assert d[2].activation_quantizer.a_bits == 4 and d[2].weight_quantizer.w_bits == 4
    assert list(d.state_dict().keys()) == keys                      # stateless quantizers: no new keys (DF)
    w = wbwtab.prepare(copy.deepcopy(base), A=2, W=3)
    assert isinstance(w[2], wbwtab.QuantConvTranspose2d) and w[2].weight_quantizer.W == 3
    assert list(w.state_dict().keys()) == keys
    i = iao.prepare(copy.deepcopy(base))
    assert isinstance(i[2], iao.QuantConvTranspose2d)
    extra = set(i.state_dict().keys()) - set(keys)
    assert {"2.activation_quantizer.scale", "2.weight_quantizer.scale", "2.weight_quantizer.observer.min_val"} <= extra
    assert tuple(i[2].weight_quantizer.scale.shape) == (1,)         # per-layer observers whatever q_level says (IAO:552-560)
    for m in (d[2], w[2], i[2]):                                    # geometry carried over by name
        assert m.stride == (2, 2) and m.padding == (1, 1) and m.output_padding == (0, 0) and m.groups == 1 and m.dilation == (1, 1)
        assert m.weight.shape == base[2].weight.shape and m.weight.data_ptr() == m.weight.data_ptr()
    for m in (d[2], w[2], i[2]):                                    # no CPU path: the engine refuses CPU tensors loudly
        with pytest.raises(Exception):
            m(torch.randn(1, 16, 4, 4))
