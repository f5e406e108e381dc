"""Host-side link plan of wbwtab.freeze_inference on NIN (models/nin.py) and NIN-GC: the kernel each frozen layer runs is
chosen from its shape (XNOR inside its cover, else the binary tensor-core convolution) and each hand-off takes its consumer's
format; NIN's 3 / 2 / 1 pools run on the b1 plane.  Builds and freezes on the CPU: only host-side cover queries run."""
import pytest
import torch
import torch.nn as nn

from harness import train as H


class RefConvBNReLU(nn.Module):
    """the reference nin.py block: conv, BatchNorm, ReLU and no channel_shuffle_flag"""

    def __init__(self, cin, cout, k, s=1, p=0):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, k, s, p)
        self.bn = nn.BatchNorm2d(cout)
        self.relu = nn.ReLU(inplace=True)

    def forward(self, x):
        return self.relu(self.bn(self.conv(x)))


class RefNIN(nn.Module):
    def __init__(self):
        super().__init__()
        B = RefConvBNReLU
        self.model = nn.Sequential(
            B(3, 192, 5, 1, 2), B(192, 160, 1), B(160, 96, 1), nn.MaxPool2d(3, 2, 1),
            B(96, 192, 5, 1, 2), B(192, 192, 1), B(192, 192, 1), nn.MaxPool2d(3, 2, 1),
            B(192, 192, 3, 1, 1), B(192, 192, 1), B(192, 10, 1), nn.AvgPool2d(8, 1, 0))

    def forward(self, x):
        x = self.model(x)
        return x.view(x.size(0), -1)


def _model(name, graph):
    import micronet_b200 as E
    if name == "ref_nin":
        torch.manual_seed(1)
        base = RefNIN()
    else:
        base = H.build_float_model(name, seed=1)
    if graph == "G2":
        m = E.wbwtab.prepare(base, W=3, A=2, fuse_bn=True)
    else:
        m = E.wbwtab.prepare(base, W=3, A=2, quant_inference=True)
        m = E.bn_fuse.wbwtab_model_bn_fuse(m, W=3)
        m = E.bn_fuse.wbwtab_quantize_inference_weights(m)
    return m.eval()


def _plan(m):
    import micronet_b200 as E
    return [c.__dict__.get("_mnb_frozen_plan") for c in m.modules() if isinstance(c, E.wbwtab.QuantConv2d)]


@pytest.mark.parametrize("graph", ["G2"])
@pytest.mark.parametrize("name", ["nin", "ref_nin"])
def test_nin_layers_freeze_on_b1(name, graph):
    import micronet_b200 as E
    from micronet_b200 import _lib as L
    m = _model(name, graph)
    tree = [type(k) for k in m.modules()]
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    E.wbwtab.freeze_inference(m)
    b1, bf16 = ("b1", L.XNOR_B1_PLANE), ("b1", L.XNOR_PM1_BF16)
    assert _plan(m) == [b1] * 6 + [bf16]
    pools = [k for k in m.model.children() if type(k).__name__ == "_PlanePool"]
    assert len(pools) == 2 and all((p.k, p.s, p.p) == (3, 2, 1) for p in pools)
    E.wbwtab.freeze_inference(m, enable=False)
    assert [type(k) for k in m.modules()] == tree and _plan(m) == [None] * 7
    assert all(torch.equal(v, sd[k]) for k, v in m.state_dict().items())


@pytest.mark.parametrize("graph", ["G2"])
def test_nin_gc_layers_stay_on_xnor(graph):
    import micronet_b200 as E
    from micronet_b200 import _lib as L
    m = _model("nin_gc", graph)
    E.wbwtab.freeze_inference(m)
    assert _plan(m) == [("xnor", L.XNOR_BITS)] * 6 + [("xnor", L.XNOR_PM1_BF16)]
