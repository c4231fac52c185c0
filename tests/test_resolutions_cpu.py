"""The engine's plan selection across batch sizes and resolutions, without a GPU.

``SkipAddEngine`` keeps one plan per (device, dtype).  A request [n,3,h,w] runs on the live plan when its pixels n*h*w fit
the plan's capacity (the n*h*w it was built for); otherwise a plan built for the request's own shape replaces it.
``plan_for(x, exact=True)`` (the host pipeline) needs the plan's own shape.  A stand-in ``Plan`` records what the engine
builds, and a stand-in input carries the shape of a CUDA tensor.
"""
import pytest
import torch

import models
from fastdepth_b200 import engine as fengine
from fastdepth_b200 import plan as fplan


class StandInPlan:
    built = []

    def __init__(self, n, h, w, dtype, device_index):
        self.n, self.h, self.w, self.dtype, self.device_index = n, h, w, dtype, device_index
        self.closed = False
        self.options = {}
        StandInPlan.built.append(self)

    @classmethod
    def from_module(cls, module, n, h, w, dtype, device_index):
        return cls(n, h, w, dtype, device_index)

    def set_option(self, name, value):
        self.options[name] = int(value)

    def get_option(self, name):
        return self.options.get(name, 0)

    def close(self):
        self.closed = True


class CudaLike:
    """What ``plan_for`` reads of a CUDA tensor."""

    def __init__(self, n, h, w, dtype=torch.float16, device=0):
        self.shape = torch.Size((n, 3, h, w))
        self.dtype = dtype
        self.device = torch.device('cuda', device)
        self.is_cuda = True

    def dim(self):
        return 4


@pytest.fixture
def engine(monkeypatch):
    monkeypatch.setattr(fplan, 'Plan', StandInPlan)
    StandInPlan.built = []
    m = models.MobileNetSkipAdd((64, 96), pretrained=False).eval().half()
    return fengine.SkipAddEngine(m)


def _live(eng):
    assert len(eng.plans) == 1
    p = next(iter(eng.plans.values()))
    return p.n, p.h, p.w


@pytest.mark.parametrize('seq, want', [
    # the batch-size policy at one resolution stays as it was
    ([(64, 224, 224), (14, 224, 224), (64, 224, 224)], [(64, 224, 224)] * 3),
    ([(64, 224, 224), (80, 224, 224)], [(64, 224, 224), (80, 224, 224)]),
    # 224x224 b64 (3.2 M pixels) is replaced by 480x640 b16 (4.9 M), which then serves 224x224 b64 again
    ([(64, 224, 224), (16, 480, 640), (64, 224, 224)], [(64, 224, 224), (16, 480, 640), (16, 480, 640)]),
    # smaller and other-shaped requests that fit never replace the plan
    ([(16, 480, 640), (8, 480, 640), (32, 256, 320), (64, 64, 96), (1, 32, 32), (2, 32, 64), (97, 224, 224)],
     [(16, 480, 640)] * 7),
    # exactly the capacity in pixels fits; one image more does not
    ([(4, 224, 224), (1, 448, 448), (4, 224, 448)], [(4, 224, 224), (4, 224, 224), (4, 224, 448)]),
    # a larger image at batch 1 replaces a plan whose batch was larger but whose pixels were fewer
    ([(8, 64, 96), (1, 480, 640)], [(8, 64, 96), (1, 480, 640)]),
])
def test_plan_kept_or_replaced(engine, seq, want):
    for shape, live in zip(seq, want):
        p = engine.plan_for(CudaLike(*shape))
        assert (p.n, p.h, p.w) == live, (shape, live)
        assert _live(engine) == live
    assert len(StandInPlan.built) == len(set(want))


def test_one_plan_per_dtype_and_device(engine):
    engine.plan_for(CudaLike(64, 224, 224))
    engine.plan_for(CudaLike(16, 480, 640, device=1))
    assert sorted(engine.plans) == [(0, torch.float16), (1, torch.float16)]
    assert engine.plans[(0, torch.float16)].n == 64 and engine.plans[(1, torch.float16)].n == 16


def test_exact_needs_the_plan_shape(engine):
    big = engine.plan_for(CudaLike(16, 480, 640))
    assert engine.plan_for(CudaLike(16, 480, 640), exact=True) is big
    # the host pipeline moves the plan's whole (N, H, W): a request that merely fits gets a plan of its own shape
    p = engine.plan_for(CudaLike(64, 224, 224), exact=True)
    assert p is not big and (p.n, p.h, p.w) == (64, 224, 224) and _live(engine) == (64, 224, 224)
    p2 = engine.plan_for(CudaLike(64, 224, 224), exact=True)
    assert p2 is p
    p3 = engine.plan_for(CudaLike(32, 224, 224), exact=True)   # same pixels per image, fewer images: still its own plan
    assert (p3.n, p3.h, p3.w) == (32, 224, 224)
    p4 = engine.plan_for(CudaLike(32, 224, 448), exact=True)   # the same pixels, another shape
    assert (p4.n, p4.h, p4.w) == (32, 224, 448)
    # and the non-exact path keeps running on whatever is live while it fits
    assert engine.plan_for(CudaLike(8, 224, 224)) is p4


def test_refresh_and_options_reach_the_one_plan(engine):
    p = engine.plan_for(CudaLike(64, 224, 224))
    engine.set_option('chain', 0)
    assert p.options['chain'] == 0
    q = engine.plan_for(CudaLike(16, 480, 640))
    assert q is not p and q.options['chain'] == 0              # options carry over to the replacing plan
    engine.refresh()
    assert q.closed and engine.plans == {}


def test_resolution_rules_still_raise(engine):
    with pytest.raises(RuntimeError, match='multiples of 32'):
        engine.plan_for(CudaLike(1, 224, 200))
    assert engine.plans == {}
