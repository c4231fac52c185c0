"""GPU parity tests: the CUDA path (through models.MobileNetSkipAdd -> ctypes -> C-ABI) against the
oracle and the committed golden vectors.  Tolerances are north_star's: 1e-3 relative for fp32,
1e-2 for fp16, both against the reference forward evaluated in fp32 (golden vectors from the live
reference, or the pinned oracle on the same storage-dtype-representable parameters and inputs).
bf16, which north_star does not bound, is checked at 1e-1 element-wise (8 mantissa bits: the same
storage roundings emulated on the CPU give 3.5e-2 on these weights; the reference run in bf16
against itself in fp32 shows 6.5e-2, BASELINE.md section 3) plus a delta1/RMSE agreement check.
The synthetic weights are conditioned so that the numbers mean something: see
fastdepth_b200/synthetic.py (a random BN+ReLU net is otherwise chaotic and even the reference's own
fp16 forward is 2-9 % away from its fp32 forward)."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, rel_err, storage_emulated_forward
from fastdepth_b200 import synthetic

pytestmark = pytest.mark.gpu

TOL = {torch.float32: 1e-3, torch.float16: 1e-2, torch.bfloat16: 1e-1}
# intermediate tensors (bug localisation only): the 2 % 'hot' BN channels (gamma up to 3.5) amplify the
# storage noise of single elements ~4x before the next layers average it out again; worst measured: 6.2e-2 on one
# element of the pruned net's 3x2-pixel conv12 map (the END-TO-END bound above is the contract and is not relaxed)
STAGE_TOL = {torch.float32: 1e-3, torch.float16: 8e-2, torch.bfloat16: 3e-1}


def oracle():
    from oracle import fastdepth_oracle as orc
    return orc


# against the storage-emulated oracle (conftest.storage_emulated_forward: same fp16/bf16 rounding points as the kernels)
# only accumulation order and one-ulp rounding flips remain; flips propagate like fresh storage noise through the deep
# stages, so a single stage gets 2e-2 (fp16, calm recipe) -- 4x sharper than the 8e-2 the hot recipe needs against plain
# fp32 -- and the END-TO-END bound stays 1e-2
EMUL_STAGE_TOL = {('calm', torch.float16): 2e-2, ('calm', torch.bfloat16): 1.5e-1,
                  ('hot', torch.float16): 5e-2, ('hot', torch.bfloat16): 3e-1}
EMUL_FINAL_TOL = {torch.float16: 1e-2, torch.bfloat16: 8e-2}


def make_model(widths, dtype, hw=(224, 224), seed=1, recipe='hot'):
    import models
    sd = synthetic.synthetic_state_dict(widths, seed=seed, recipe=recipe)
    m = models.MobileNetSkipAdd(hw, pretrained=False, widths=widths)
    m.load_state_dict(sd)
    return m.eval().cuda().to(dtype), sd


def quantised_sd(sd, dtype):
    """What the reference sees after model.half(): parameters rounded to the storage dtype."""
    if dtype == torch.float32:
        return sd
    return {k: (v.to(dtype).float() if v.is_floating_point() else v) for k, v in sd.items()}


def run(m, x, dtype, path, chain=1):
    with torch.no_grad():
        from fastdepth_b200.engine import SkipAddEngine
        eng = SkipAddEngine(m)
        eng.set_option('path', path)
        eng.set_option('chain', chain)
        m.__dict__['_fd_engine'] = eng
        y = m(x.cuda().to(dtype))
    torch.cuda.synchronize()
    return y, eng


@pytest.mark.parametrize('name', ['skipadd_stock_2x64x96', 'skipadd_pruned_2x64x96', 'skipadd_stock_1x224x224'])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize('path', [0, 1])
def test_golden_end_to_end(name, dtype, path):
    fx = np.load(os.path.join(GOLDEN, name + '.npz'))
    widths = (tuple(int(v) for v in fx['widths_enc']), tuple(int(v) for v in fx['widths_dec']))
    n, h, w = (int(v) for v in fx['shape'])
    m, _ = make_model(widths, dtype, (h, w), seed=int(fx['wseed']))
    x = synthetic.synthetic_input(n, h, w, seed=int(fx['xseed']))
    y, _ = run(m, x, dtype, path)
    want = torch.from_numpy(fx['output'])
    assert y.shape == want.shape and y.dtype == dtype and y.is_contiguous()
    assert (want == 0).float().mean() < 0.5
    assert rel_err(y.float().cpu(), want) <= TOL[dtype]


@pytest.mark.parametrize('widths', [synthetic.STOCK_WIDTHS, synthetic.PRUNED_WIDTHS], ids=['stock', 'pruned'])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('path', [0, 1])
@pytest.mark.parametrize('fold', [0, 1])
def test_stage_by_stage(widths, dtype, path, fold):
    """Every named child's output vs the oracle (localises the first diverging stage)."""
    orc = oracle()
    m, sd = make_model(widths, dtype, (96, 64))
    x = synthetic.synthetic_input(3, 96, 64, seed=4)
    from fastdepth_b200.engine import SkipAddEngine
    eng = SkipAddEngine(m)
    eng.set_option('path', path)
    eng.set_option('fold_head', fold)
    eng.set_option('inplace_skip', 0)          # keep every stage buffer inspectable (skip sources are not overwritten)
    eng.set_option('chain', 0)                 # ... and every stage materialised (no multi-layer chain kernel)
    eng.set_option('tma_epilogue', fold)       # fold=0 runs also exercise the LSU epilogue of the fused blocks
    m.__dict__['_fd_engine'] = eng
    with torch.no_grad():
        y = m(x.cuda().to(dtype))
    torch.cuda.synchronize()
    stages = {}
    want = orc.skipadd_forward(quantised_sd(sd, dtype), x.to(dtype).float(), stages=stages)
    plan = next(iter(eng.plans.values()))
    for i, name in enumerate(plan.names[:-1]):
        got = plan.stage_tensor(i).float().cpu().permute(0, 3, 1, 2)
        ref = stages[name]
        if fold and name == 'decode_conv5':
            if path == 1 and dtype != torch.float32:
                continue                               # head fused into the block: never materialised
            ref = stages['decode_conv5.pw']            # the folded plan keeps the low-res tensor
        assert got.shape == ref.shape, name
        assert rel_err(got, ref) <= STAGE_TOL[dtype], name
    assert rel_err(y.float().cpu(), want) <= TOL[dtype]


@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16])
def test_full_size_batch64_properties(dtype):
    """BASELINE metric config (N=64, 224x224): oracle on a few images + size-independent properties:
    images are independent (a batch equals its images run alone, bit-exact) and the fused path
    agrees with the unfused one."""
    orc = oracle()
    m, sd = make_model(synthetic.STOCK_WIDTHS, dtype)
    x = synthetic.synthetic_input(64, 224, 224, seed=9)
    y1, _ = run(m, x, dtype, 1)
    y0, _ = run(m, x, dtype, 0)
    assert rel_err(y1.float().cpu(), y0.float().cpu()) <= TOL[dtype]
    pick = [0, 31, 63]
    want = orc.skipadd_forward(quantised_sd(sd, dtype), x[pick].to(dtype).float())
    assert rel_err(y1[pick].float().cpu(), want) <= TOL[dtype]
    ys, _ = run(m, x[pick], dtype, 1)
    assert torch.equal(ys, y1[pick])
    assert torch.isfinite(y1.float()).all()


def test_bf16_metric_agreement():
    """config 4 is bf16; north_star gives no element-wise bf16 bound, so delta1/RMSE agreement is the
    binding check (BASELINE.md section 3)."""
    orc = oracle()
    m, sd = make_model(synthetic.STOCK_WIDTHS, torch.bfloat16)
    x = synthetic.synthetic_input(8, 224, 224, seed=2)
    y, _ = run(m, x, torch.bfloat16, 1)
    ref = orc.skipadd_forward(sd, x)
    tgt = synthetic.synthetic_target(ref, seed=1)
    a, _ = orc.average_per_image(y.float().cpu().numpy(), tgt.numpy())
    b, _ = orc.average_per_image(ref.numpy(), tgt.numpy())
    assert abs(a['delta1'] - b['delta1']) < 0.02
    assert abs(a['rmse'] - b['rmse']) / b['rmse'] < 0.05


def test_non_contiguous_input_and_high_res():
    orc = oracle()
    m, sd = make_model(synthetic.STOCK_WIDTHS, torch.float16, (480, 640))
    x = synthetic.synthetic_input(2, 480, 640, seed=3)
    xt = x.permute(0, 1, 3, 2).contiguous().permute(0, 1, 3, 2)      # same values, exotic strides
    assert not xt.is_contiguous()
    y, _ = run(m, xt, torch.float16, 1)
    want = orc.skipadd_forward(quantised_sd(sd, torch.float16), x.half().float())
    assert rel_err(y.float().cpu(), want) <= 1e-2


def test_error_behaviour():
    m, _ = make_model(synthetic.STOCK_WIDTHS, torch.float16)
    with pytest.raises(RuntimeError):                      # reference: size mismatch at the first skip add
        m(torch.rand(1, 3, 228, 304, device='cuda', dtype=torch.float16))
    with pytest.raises(RuntimeError, match='should be the same'):
        m(torch.rand(1, 3, 64, 64, device='cuda', dtype=torch.float32))
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        m(torch.rand(1, 3, 64, 64).half())


def test_weight_update_is_picked_up():
    m, sd = make_model(synthetic.STOCK_WIDTHS, torch.float32, (64, 64))
    x = synthetic.synthetic_input(1, 64, 64, seed=1).cuda()
    with torch.no_grad():
        a = m(x).clone()
        m.load_state_dict(synthetic.synthetic_state_dict(seed=5))
        b = m(x)
    want = oracle().skipadd_forward(synthetic.synthetic_state_dict(seed=5), x.cpu())
    assert not torch.allclose(a, b) and rel_err(b.cpu(), want) <= 1e-3


def test_metrics_kernel_known_answer():
    from fastdepth_b200 import evaluate, plan
    fx = np.load(os.path.join(GOLDEN, 'metrics_known_answer.npz'))
    names = [str(n) for n in fx['names']]
    sums = evaluate.new_sums('cuda')
    plan.metrics_accumulate(torch.from_numpy(fx['multi_out']).cuda(), torch.from_numpy(fx['multi_tgt']).cuda(), sums)
    avg = evaluate.finalize(sums)
    assert avg['count'] == 3
    for k, v in zip(names, fx['multi_avg']):
        assert avg[k] == pytest.approx(float(v), rel=5e-5), k
    sums.zero_()
    p = torch.from_numpy(fx['pred_sub4']).cuda().view(1, 1, 56, 56)
    t = torch.from_numpy(fx['depth_sub4']).cuda().view(1, 1, 56, 56)
    plan.metrics_accumulate(p, t, sums)
    one = evaluate.finalize(sums)
    for k, v in zip(names, fx['sub4_values']):
        assert one[k] == pytest.approx(float(v), rel=5e-5), k


def test_sharded_evaluate_single_gpu():
    from fastdepth_b200 import evaluate
    orc = oracle()
    m, sd = make_model(synthetic.STOCK_WIDTHS, torch.float32, (64, 96))
    x = synthetic.synthetic_input(6, 64, 96, seed=8)
    ref = orc.skipadd_forward(sd, x)
    tgt = synthetic.synthetic_target(ref, seed=2)
    got = evaluate.evaluate(m, [(x[:4], tgt[:4]), (x[4:], tgt[4:])], torch.device('cuda:0'))
    want, n = orc.average_per_image(ref.numpy(), tgt.numpy())
    assert got['count'] == n
    for k in ('rmse', 'mae', 'delta1', 'absrel', 'lg10'):
        assert got[k] == pytest.approx(want[k], rel=2e-3, abs=1e-4), k
    # several batches in flight (three plan copies on their own streams, one sum vector per lane): the same sums, bit for bit
    batches = [(x[i:i + 1], tgt[i:i + 1]) for i in range(6)]
    _, s1 = evaluate.evaluate(m, batches, torch.device('cuda:0'), return_sums=True)
    _, s3 = evaluate.evaluate(m, batches, torch.device('cuda:0'), return_sums=True, lanes=3)
    assert torch.equal(s1, s3)


def test_pipeline_api_matches_forward():
    """fd_pipeline_submit / fd_pipeline_wait (host buffers, 3 batches in flight) == fd_forward per batch."""
    m, sd = make_model(synthetic.STOCK_WIDTHS, torch.float16, (64, 96))
    from fastdepth_b200.engine import SkipAddEngine
    eng = SkipAddEngine(m)
    xs = [synthetic.synthetic_input(4, 64, 96, seed=20 + i).half() for i in range(7)]
    plan = eng.plan_for(xs[0].cuda())
    want = []
    with torch.no_grad():
        for x in xs:
            y = torch.empty((4, 1, 64, 96), dtype=torch.float16, device='cuda')
            plan.forward(x.cuda(), y, torch.cuda.current_stream().cuda_stream)
            want.append(y.cpu())
    torch.cuda.synchronize()
    xh = [x.pin_memory() for x in xs]
    yh = [torch.empty((4, 1, 64, 96), dtype=torch.float16).pin_memory() for _ in xs]
    tickets = [plan.pipeline_submit(a, b) for a, b in zip(xh, yh)]
    assert tickets == list(range(len(xs)))
    for t in reversed(tickets):
        plan.pipeline_wait(t)
    for a, b in zip(yh, want):
        assert torch.equal(a, b)
    y2 = torch.empty((4, 1, 64, 96), dtype=torch.float16).pin_memory()
    plan.forward_host(xh[3], y2, torch.cuda.current_stream().cuda_stream)
    assert torch.equal(y2, want[3])


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
def test_mobilenet_nnconv5dw_no_skips(dtype):
    """SURVEY.md section 8f row 2: models.MobileNet(decoder='nnconv5dw') takes the same fused path (no skips)."""
    import models
    fx = np.load(os.path.join(GOLDEN, 'nnconv5dw_stock_2x64x96.npz'))
    n, h, w = (int(v) for v in fx['shape'])
    sd = synthetic.to_mobilenet_keys(synthetic.synthetic_state_dict(seed=int(fx['wseed'])))
    m = models.MobileNet('nnconv5dw', (h, w), pretrained=False)
    m.load_state_dict(sd)
    m = m.eval().cuda().to(dtype)
    x = synthetic.synthetic_input(n, h, w, seed=int(fx['xseed']))
    with torch.no_grad():
        y = m(x.cuda().to(dtype))
    torch.cuda.synchronize()
    assert '_fd_engine' in m.__dict__                      # really went through the C-ABI, not PyTorch eager
    assert rel_err(y.float().cpu(), torch.from_numpy(fx['output'])) <= TOL[dtype]
    # the dense 5x5 decoder is not a kernel target: it stays on stock PyTorch
    md = models.MobileNet('nnconv5', (h, w), pretrained=False).eval().cuda()
    with torch.no_grad():
        assert md(x.cuda()).shape == (n, 1, h, w) and '_fd_engine' not in md.__dict__


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('path', [0, 1])
def test_skipconcat(dtype, path):
    """SURVEY.md section 8f row 1: MobileNetSkipConcat -- both halves of every concatenation are channel-slice writes
    into one wide NHWC buffer (TMA stores with a row pitch on path 1, pitched LSU stores on path 0)."""
    import models
    orc = oracle()
    fx = np.load(os.path.join(GOLDEN, 'skipconcat_stock_2x64x96.npz'))
    n, h, w = (int(v) for v in fx['shape'])
    sd = synthetic.synthetic_state_dict(seed=int(fx['wseed']), skip='concat')
    m = models.MobileNetSkipConcat((h, w), pretrained=False)
    m.load_state_dict(sd)
    m = m.eval().cuda().to(dtype)
    x = synthetic.synthetic_input(n, h, w, seed=int(fx['xseed']))
    y, eng = run(m, x, dtype, path)
    assert rel_err(y.float().cpu(), torch.from_numpy(fx['output'])) <= TOL[dtype]
    y, eng = run(m, x, dtype, path, chain=0)               # every stage materialised for the stage-wise check
    assert rel_err(y.float().cpu(), torch.from_numpy(fx['output'])) <= TOL[dtype]
    # stage-wise: the decoder slices and the re-pointed skip sources
    stages = {}
    orc.skipconcat_forward(quantised_sd(sd, dtype), x.to(dtype).float(), stages=stages)
    plan = next(iter(eng.plans.values()))
    for i, name in enumerate(plan.names[:-2]):
        got = plan.stage_tensor(i).float().cpu().permute(0, 3, 1, 2)
        assert got.shape == stages[name].shape, name
        assert rel_err(got, stages[name]) <= STAGE_TOL[dtype], name
    # larger problem, many items per CTA
    x8 = synthetic.synthetic_input(8, 224, 224, seed=3)
    m2 = models.MobileNetSkipConcat((224, 224), pretrained=False)
    m2.load_state_dict(sd)
    m2 = m2.eval().cuda().to(dtype)
    y8, _ = run(m2, x8, dtype, path)
    want = orc.skipconcat_forward(quantised_sd(sd, dtype), x8[[0, 7]].to(dtype).float())
    assert rel_err(y8[[0, 7]].float().cpu(), want) <= TOL[dtype]


@pytest.mark.parametrize('widths', [synthetic.STOCK_WIDTHS, synthetic.PRUNED_WIDTHS], ids=['stock', 'pruned'])
def test_epilogue_organisations_and_item_shapes_agree_bitwise(widths, monkeypatch):
    """The planner's choices are scheduling only: output-channel splits, clusters, depthwise teams, sleeping vs spinning
    waits must all produce the SAME bits (224x224 so that every block has
    many items; the planner knobs are environment variables read when a plan is built)."""
    from fastdepth_b200.engine import SkipAddEngine
    m, _ = make_model(widths, torch.float16, (224, 224))
    x = synthetic.synthetic_input(64, 224, 224, seed=11).cuda().half()     # the metric batch: only there does the planner
    outs, kernels = [], []
    knobs = ('FD_TC_MAX_NCTA', 'FD_TC_CLUSTER', 'FD_TC_WMC', 'FD_TC_DW_TEAMS')
    for env, opts in (({}, {}),
                      ({'FD_TC_MAX_NCTA': '64', 'FD_TC_CLUSTER': '1'}, {}),
                      ({'FD_TC_MAX_NCTA': '64'}, {'wait_sleep_ns': 200}),
                      ({'FD_TC_CLUSTER': '1'}, {}),                # never a cluster
                      ({'FD_TC_CLUSTER': '1', 'FD_TC_WMC': '2'}, {}),      # weight-multicast clusters of 2 tiles
                      ({'FD_TC_CLUSTER': '1', 'FD_TC_WMC': '4'}, {}),      # ... of 4 tiles
                      ({'FD_TC_DW_TEAMS': '1'}, {}),               # eight depthwise warps in lock-step everywhere
                      ({'FD_TC_DW_TEAMS': '2'}, {})):              # two depthwise teams wherever even ring depths fit
        for k in knobs:
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        eng = SkipAddEngine(m)
        eng.set_option('chain', 0)                 # this test is about the per-block kernel's planner (conv7..11 included)
        for k, v in opts.items():
            eng.set_option(k, v)
        m.__dict__['_fd_engine'] = eng
        with torch.no_grad():
            outs.append(m(x).clone())
        kernels.append(' '.join(s['kernel'] for s in next(iter(eng.plans.values())).steps()))
    torch.cuda.synchronize()
    assert kernels[0] != kernels[1] and kernels[0] != kernels[2], kernels[2]
    assert ',cl' not in kernels[1] and ',cl' not in kernels[3], kernels[3]
    assert ',wmc2' in kernels[4] and ',wmc4' in kernels[5], (kernels[4], kernels[5])   # one weight stream multicast to a cluster
    assert ',t2' not in kernels[6] and kernels[7].count(',t2') > kernels[0].count(',t2') > 0, (kernels[0], kernels[7])
    if widths is synthetic.STOCK_WIDTHS:
        assert 'n128x4,bn128,kb8' in kernels[3] and 'n64x8,bn64,kb8' in kernels[2] and 'n128x4,bn128,kb8' not in kernels[2]   # conv7
    for i in range(1, len(outs)):
        d = (outs[0].float() - outs[i].float()).abs().max().item()
        assert d == 0.0, (i, d, kernels[i])


@pytest.mark.parametrize('widths', [synthetic.STOCK_WIDTHS, synthetic.PRUNED_WIDTHS], ids=['stock', 'pruned'])
def test_tile_sharing_clusters_agree_bitwise(widths, monkeypatch):
    """Tile-sharing clusters (2 / 4 CTAs split one tile's depthwise half and output channels, operand tiles handed over through
    DSMEM) against the cluster-less plan, forced wherever a block admits them (one wave: batch 8), stage by stage, bit for bit."""
    from fastdepth_b200.engine import SkipAddEngine
    m, _ = make_model(widths, torch.float16, (224, 224))
    x = synthetic.synthetic_input(8, 224, 224, seed=12).cuda().half()
    ref = None
    for cl in ('1', '2', '4'):
        monkeypatch.setenv('FD_TC_CLUSTER', cl)
        eng = SkipAddEngine(m)
        for k, v in (('chain', 0), ('inplace_skip', 0), ('fold_head', 0)):
            eng.set_option(k, v)
        m.__dict__['_fd_engine'] = eng
        with torch.no_grad():
            y = m(x).clone()
        plan = next(iter(eng.plans.values()))
        kern = ' '.join(s['kernel'] for s in plan.steps())
        outs = [plan.stage_tensor(i).clone() for i in range(len(plan.names) - 1)] + [y]
        torch.cuda.synchronize()
        if ref is None:
            ref = outs
            assert ',cl' not in kern, kern
            continue
        assert kern.count(',cl%s' % cl) >= 3, kern
        for i, (a, b) in enumerate(zip(ref, outs)):
            assert torch.equal(a, b), (cl, i, kern)


def test_forward_lanes_match_the_module_forward():
    """fastdepth_b200.engine.ForwardLanes (three plan copies on their own streams, batches round-robin) returns, for every batch,
    the bits the module's own forward returns; the host pipeline of the lanes too."""
    from fastdepth_b200.engine import ForwardLanes
    m, _ = make_model(synthetic.STOCK_WIDTHS, torch.float16, (64, 96))
    xs = [synthetic.synthetic_input(3, 64, 96, seed=40 + i).cuda().half() for i in range(7)]
    with torch.no_grad():
        want = [m(x).clone() for x in xs]
    lanes = ForwardLanes(m, lanes=3)
    outs = [lanes.forward(x) for x in xs]
    for (y, done), w in zip(outs, want):
        done.synchronize()
        assert torch.equal(y, w)
    xh = [x.cpu().pin_memory() for x in xs]
    yh = [torch.empty((3, 1, 64, 96), dtype=torch.float16).pin_memory() for _ in xs]
    handles = [lanes.submit(a, b, xs[0]) for a, b in zip(xh, yh)]
    for hnd in handles:
        lanes.wait(hnd)
    for b, w in zip(yh, want):
        assert torch.equal(b, w.cpu())
    lanes.synchronize()


def test_one_plan_on_two_streams_is_ordered_not_corrupted():
    """ADVICE r1: a plan owns one set of activation buffers.  Forwards enqueued on two different streams without any
    synchronisation in between must come out as if they had run one after the other."""
    from fastdepth_b200.engine import SkipAddEngine
    m, _ = make_model(synthetic.STOCK_WIDTHS, torch.float16, (224, 224))
    xs = [synthetic.synthetic_input(16, 224, 224, seed=70 + i).cuda().half() for i in range(4)]
    with torch.no_grad():
        want = [m(x).clone() for x in xs]
    torch.cuda.synchronize()
    eng = SkipAddEngine(m)
    plan = eng.plan_for(xs[0])
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    ys = [torch.empty_like(w) for w in want]
    for rep in range(3):
        for i, x in enumerate(xs):
            plan.forward(x, ys[i], (s1 if i % 2 == 0 else s2).cuda_stream)
    torch.cuda.synchronize()
    for y, w in zip(ys, want):
        assert torch.equal(y, w)


def test_option_validation():
    from fastdepth_b200.engine import SkipAddEngine
    m, _ = make_model(synthetic.STOCK_WIDTHS, torch.float16, (64, 96))
    eng = SkipAddEngine(m)
    eng.plan_for(synthetic.synthetic_input(1, 64, 96).cuda().half())
    with pytest.raises(RuntimeError):
        eng.set_option('wait_sleep_ns', -1)
    with pytest.raises(RuntimeError):
        eng.set_option('graph', 2)
    with pytest.raises(RuntimeError):
        eng.set_option('no_such_option', 1)


@pytest.mark.parametrize('widths', [synthetic.STOCK_WIDTHS, synthetic.PRUNED_WIDTHS], ids=['stock', 'pruned'])
@pytest.mark.parametrize('recipe', ['calm', 'hot'])
@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16])
def test_stage_by_stage_vs_storage_emulated_oracle(widths, recipe, dtype):
    """Sharper stage-wise check (VERDICT r1 'harden parity'): a second, well-conditioned weight recipe without hot BN
    channels ('calm'), and every stage compared with the oracle evaluated WITH the product's storage roundings, at the
    end-to-end tolerance -- a few-percent bug in one stage can no longer hide behind the 8e-2 stage bound that plain
    fp32 comparison needs on the hot recipe.  Also pins the calm recipe's plain-fp32 distance at 2e-2."""
    m, sd = make_model(widths, dtype, (96, 64), recipe=recipe)
    x = synthetic.synthetic_input(3, 96, 64, seed=4)
    from fastdepth_b200.engine import SkipAddEngine
    eng = SkipAddEngine(m)
    eng.set_option('inplace_skip', 0)
    eng.set_option('fold_head', 0)
    eng.set_option('chain', 0)                 # every stage materialised (the chain kernel keeps conv7..10 in shared memory)
    m.__dict__['_fd_engine'] = eng
    with torch.no_grad():
        y = m(x.cuda().to(dtype))
    torch.cuda.synchronize()
    emu = {}
    want = storage_emulated_forward(sd, x, dtype, stages=emu)
    plan = next(iter(eng.plans.values()))
    worst = {}
    for i, name in enumerate(plan.names[:-1]):
        got = plan.stage_tensor(i).float().cpu().permute(0, 3, 1, 2)
        assert got.shape == emu[name].shape, name
        worst[name] = rel_err(got, emu[name])
    bad = {k: v for k, v in worst.items() if v > EMUL_STAGE_TOL[(recipe, dtype)]}
    assert not bad, bad
    assert rel_err(y.float().cpu(), want) <= EMUL_FINAL_TOL[dtype]
    if recipe == 'calm' and dtype == torch.float16:
        ref = {}
        oracle().skipadd_forward(quantised_sd(sd, dtype), x.to(dtype).float(), stages=ref)
        for i, name in enumerate(plan.names[:-1]):
            got = plan.stage_tensor(i).float().cpu().permute(0, 3, 1, 2)
            assert rel_err(got, ref[name]) <= 2.5e-2, name


CONFIGS = {   # BASELINE.json configs 2, 3, 5 at their stated batch (VERDICT r1 row +2); oracle on picked images
    'cfg2_stock_b32_224': (synthetic.STOCK_WIDTHS, 32, 224, 224, [0, 13, 31]),
    'cfg3_pruned_b64_224': (synthetic.PRUNED_WIDTHS, 64, 224, 224, [0, 31, 63]),
    'cfg5_stock_b16_480x640': (synthetic.STOCK_WIDTHS, 16, 480, 640, [0, 15]),
}


@pytest.mark.parametrize('cfg', sorted(CONFIGS))
def test_baseline_configs_vs_oracle(cfg):
    """fp16 at the configuration's full batch against the oracle (1e-2, north_star) on picked images, plus the
    size-independent property that the picked images run alone give the same bits."""
    widths, n, h, w, pick = CONFIGS[cfg]
    orc = oracle()
    dtype = torch.float16
    m, sd = make_model(widths, dtype, (h, w))
    x = synthetic.synthetic_input(n, h, w, seed=21)
    y, eng = run(m, x, dtype, 1)
    assert y.shape == (n, 1, h, w) and torch.isfinite(y.float()).all()
    want = orc.skipadd_forward(quantised_sd(sd, dtype), x[pick].to(dtype).float())
    assert (want == 0).float().mean() < 0.5
    assert rel_err(y[pick].float().cpu(), want) <= TOL[dtype]
    ys, _ = run(m, x[pick], dtype, 1)
    assert torch.equal(ys, y[pick])
    kernels = ' '.join(s['kernel'] for s in next(iter(eng.plans.values())).steps())
    assert 'block_tc' in kernels or 'chain_tc' in kernels, kernels          # the fused tensor-core path really ran


def test_bf16_elementwise_against_storage_emulated_oracle():
    """config 4's dtype: element-wise against the oracle WITH bf16 storage roundings (what any bf16 implementation of
    the reference computes) -- tighter than the 1e-1 bound against un-rounded fp32."""
    m, sd = make_model(synthetic.STOCK_WIDTHS, torch.bfloat16)
    x = synthetic.synthetic_input(4, 224, 224, seed=5)
    y, _ = run(m, x, torch.bfloat16, 1)
    want = storage_emulated_forward(sd, x, torch.bfloat16)
    assert rel_err(y.float().cpu(), want) <= 4e-2


def test_validate_loop_drops_in():
    """The reference's only caller, main.validate (main.py:63-127), restated on synthetic (input, target) pairs: a
    whole-module pickle is loaded the way main.py:49-57 does, ``model.eval()``, batch-size-1 loader, ``input.cuda()``,
    ``pred = model(input)`` under no_grad, a per-image Result.evaluate on ``pred.data`` weighted by ``input.size(0)``
    (AverageMeter, metrics.py:71-95), and ``pred.data.cpu().numpy()`` as utils.merge_into_row reads it (utils.py:46-49).
    The averages must equal the oracle's forward + the oracle's per-image metrics."""
    import io
    import models
    orc = oracle()
    sd = synthetic.synthetic_state_dict(seed=3)
    m0 = models.MobileNetSkipAdd((64, 96), pretrained=False)
    m0.load_state_dict(sd)
    buf = io.BytesIO()
    torch.save({'model': m0, 'epoch': 7}, buf)                 # what train() writes, main.py / utils.save_checkpoint
    buf.seek(0)
    checkpoint = torch.load(buf, weights_only=False)
    model = checkpoint['model'] if type(checkpoint) is dict else checkpoint
    model = model.cuda()
    xs = synthetic.synthetic_input(5, 64, 96, seed=31)
    ref = orc.skipadd_forward(sd, xs)
    tgts = synthetic.synthetic_target(ref, seed=4)
    val_loader = [(xs[i:i + 1], tgts[i:i + 1]) for i in range(5)]

    sums, count, merged = {}, 0, []
    model.eval()
    for i, (input, target) in enumerate(val_loader):
        input, target = input.cuda(), target.cuda()
        with torch.no_grad():
            pred = model(input)
        result = orc.evaluate_one(pred.data.cpu().numpy(), target.data.cpu().numpy())
        n = input.size(0)
        for k, v in result.items():
            sums[k] = sums.get(k, 0.0) + n * v
        count += n
        merged.append(np.squeeze(pred.data.cpu().numpy()))
    avg = {k: v / count for k, v in sums.items()}
    want, n_img = orc.average_per_image(ref.numpy(), tgts.numpy())
    assert count == n_img == 5 and merged[0].shape == (64, 96)
    for k in ('rmse', 'mae', 'delta1', 'absrel', 'lg10', 'irmse'):
        assert avg[k] == pytest.approx(want[k], rel=2e-3, abs=1e-4), k
    assert '_fd_engine' in model.__dict__                     # the forward went through the C-ABI


def test_inplace_edit_of_an_inner_layer_is_picked_up():
    """engine freshness: an in-place write to ANY parameter (not just conv0 / the head BN) re-packs the weights."""
    m, sd = make_model(synthetic.STOCK_WIDTHS, torch.float32, (64, 64))
    x = synthetic.synthetic_input(1, 64, 64, seed=1).cuda()
    with torch.no_grad():
        a = m(x).clone()
        m.conv7[3].weight.mul_(1.5)
        m.decode_conv2[0][1].running_var.mul_(0.5)
        b = m(x)
    sd2 = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    want = oracle().skipadd_forward(sd2, x.cpu())
    assert not torch.allclose(a, b) and rel_err(b.cpu(), want) <= 1e-3


def test_two_plans_with_different_options_do_not_share_launch_state():
    """ADVICE r1: pdl / wait_sleep_ns live in each kernel plan, not in process globals."""
    from fastdepth_b200.engine import SkipAddEngine
    m, _ = make_model(synthetic.STOCK_WIDTHS, torch.float16, (64, 96))
    x = synthetic.synthetic_input(2, 64, 96, seed=2).cuda().half()
    e1, e2 = SkipAddEngine(m), SkipAddEngine(m)
    e1.set_option('pdl', 1)
    e2.set_option('pdl', 0)
    e2.set_option('wait_sleep_ns', 300)
    outs = []
    with torch.no_grad():
        for e in (e1, e2, e1, e2):
            outs.append(e(x).clone())
    torch.cuda.synchronize()
    assert all(torch.equal(outs[0], o) for o in outs[1:])


@pytest.mark.parametrize('widths', [synthetic.STOCK_WIDTHS, synthetic.PRUNED_WIDTHS], ids=['stock', 'pruned'])
@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16])
@pytest.mark.parametrize('shape', [(3, 96, 64), (2, 64, 96), (5, 224, 224), (80, 224, 224)], ids=lambda s: '%dx%dx%d' % s)
def test_chain_kernel_matches_per_layer_kernels(widths, dtype, shape):
    """conv7..conv11 as ONE 2-CTA-cluster kernel (activations resident in shared memory, wgmma in passes of 128 channels) against the
    same five blocks run layer by layer by the per-block kernel: the chain's output tensor (conv11) and the final depth map,
    on 4x6 / 6x4 / 14x14 maps, odd image counts and more images than clusters, stock and pruned (K and N not multiples of
    64) widths.  Both paths round at the same points, so they agree to accumulation order; each is also held to the oracle."""
    n, h, w = shape
    m, sd = make_model(widths, dtype, (h, w))
    x = synthetic.synthetic_input(n, h, w, seed=17)
    y1, e1 = run(m, x, dtype, 1, chain=1)
    p1 = next(iter(e1.plans.values()))
    kern = [s['kernel'] for s in p1.steps()]
    assert any('chain_tc' in k for k in kern), kern
    c11 = p1.names.index('conv11')
    a = p1.stage_tensor(c11).float().cpu().clone()
    y0, e0 = run(m, x, dtype, 1, chain=0)
    p0 = next(iter(e0.plans.values()))
    assert not any('chain_tc' in s['kernel'] for s in p0.steps())
    b = p0.stage_tensor(c11).float().cpu()
    tol = 4e-3 if dtype == torch.float16 else 3e-2
    assert rel_err(a, b) <= tol
    assert rel_err(y1.float().cpu(), y0.float().cpu()) <= tol
    pick = sorted({0, n // 2, n - 1})
    want = oracle().skipadd_forward(quantised_sd(sd, dtype), x[pick].to(dtype).float())
    assert rel_err(y1[pick].float().cpu(), want) <= TOL[dtype]
    ys, _ = run(m, x[pick], dtype, 1, chain=1)             # images are independent: same bits alone as in the batch
    assert torch.equal(ys, y1[pick])
