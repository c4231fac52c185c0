import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a real H100 (run with -m gpu on a machine that has one)')


@pytest.fixture(scope='session')
def built_lib():
    """The in-tree shared library (built on demand; nvcc cross-compiles without a GPU)."""
    from fastdepth_b200 import build
    from oracle import build_oracle
    build_oracle.build()                      # the plain-C oracle primitives ride along (gcc, test infrastructure)
    return build.build()


def rel_err(got, want):
    """max |got-want| / max(|want|, mean|want|): element-wise relative error with a floor at the
    tensor's mean magnitude, so exact zeros after ReLU do not blow the ratio up (SURVEY.md 7.4.7)."""
    import torch
    got = got.double(); want = want.double()
    denom = torch.maximum(want.abs(), want.abs().mean())
    return ((got - want).abs() / denom).max().item()


def storage_emulated_forward(sd, x, dtype, stages=None):
    """The oracle's forward with the PRODUCT's storage roundings: every tensor that the CUDA path keeps in the 16-bit
    storage dtype (stem output, each depthwise result, each pointwise result, each skip sum, the final map) is rounded
    to that dtype, all arithmetic stays fp32 (oracle primitives).  Against this the kernels may differ only by
    accumulation order and by one-ulp rounding flips that propagate -- an order of magnitude tighter than comparing
    with the un-rounded fp32 forward, whose distance from ANY 16-bit implementation is dominated by storage noise
    (1.2e-2 on the 'calm' synthetic recipe, 3-5e-2 on the 'hot' one, measured on the CPU with this very function)."""
    import torch
    from oracle import fastdepth_oracle as orc
    f = torch.float32

    def q(t):
        return t.to(dtype).float()
    sdq = {k: (v.to(dtype).float() if v.is_floating_point() else v) for k, v in sd.items()}
    x = q(x)
    keep = {}
    x = q(orc.stem(x, sdq, f))
    if stages is not None:
        stages['conv0'] = x
    for i in range(1, 14):
        x = q(orc.encoder_pw(q(orc.encoder_dw(x, sdq, i, f)), sdq, i, f))
        if stages is not None:
            stages['conv%d' % i] = x
        if i in (1, 3, 5):
            keep[i] = x
    add_after = {4: 1, 3: 3, 2: 5}
    for j in range(1, 6):
        p = q(orc.decoder_pw(q(orc.decoder_dw(x, sdq, j, f)), sdq, j, f))
        x = orc.upsample2x(p)
        if j in add_after:
            x = q(x + keep[add_after[j]])
        if stages is not None:
            stages['decode_conv%d.pw' % j] = p
            stages['decode_conv%d' % j] = x
    x = q(orc.head(x, sdq, f))
    if stages is not None:
        stages['decode_conv6'] = x
    return x
