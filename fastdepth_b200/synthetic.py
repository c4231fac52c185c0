"""Deterministic synthetic weights and inputs for parity tests, smoke() and bench.py.

Trained FastDepth weights are download links in the reference (README.md:26-46) and there is
no network, so every measurement here uses random-init weights of the named architecture.
Plain default init collapses activations to ~1e-3 and makes relative-error parity vacuous
(SURVEY.md section 4 "synthetic-weight pitfalls"), hence this recipe:

* conv weights: encoder N(0, sqrt(2/fan_in)); decoder U(-b, b), b = 1/sqrt(fan_in) (PyTorch default,
  which the SkipAdd decoder keeps because of the ``weights_init``-on-Sequential no-op, reference
  models.py:699-704); the head's weights are made positive so the output is depth-like;
* BN: gamma ~ U(0.25, 0.75) (2 % hot channels U(2.5, 3.5)), beta ~ N(0.6, 0.25); running_mean / running_var CALIBRATED on a seeded probe
  batch (what a trained checkpoint carries) -- see ``synthetic_state_dict``;
* last BN (decode_conv6): gamma = 1, beta = 3 so the final ReLU leaves a live, metres-like map.

Random draws come from ``numpy.random.Generator(PCG64(seed))`` in a fixed order and the calibration
runs in fp64, so the fp32 values are reproducible across machines (the golden fixtures depend on it).
"""
import numpy as np
import torch

# NetAdapt-pruned widths recovered from the reference's TVM tuning log
# (tvm_compile/tuning/tx2-gpu.mobilenet-nnconv5dw-skipadd-pruned.trials=2000.stop=600.log,
#  lines 38..1 in network order; SURVEY.md section 8a-a10).
PRUNED_ENCODER = (16, 56, 88, 120, 144, 256, 408, 376, 272, 288, 296, 328, 480, 512)
PRUNED_DECODER = (200, 256, 120, 56, 16)
PRUNED_WIDTHS = (PRUNED_ENCODER, PRUNED_DECODER)

STOCK_ENCODER = (32, 64, 128, 128, 256, 256, 512, 512, 512, 512, 512, 512, 1024, 1024)
STOCK_DECODER = (512, 256, 128, 64, 32)
STOCK_WIDTHS = (STOCK_ENCODER, STOCK_DECODER)


_CACHE = {}


# Conditioning knobs, tuned in round 1 (see DESIGN.md 'synthetic weights'): a random BN+ReLU network is
# chaotic for E[gamma^2] >~ 1 -- the reference's OWN fp16 forward then differs from its fp32 forward by
# 2-9 % and a 1e-2 criterion is noise.  With these values the fp16 storage noise reaches the output at
# ~4e-3 max / 7e-4 mean while a 5 % weight error in conv7 still moves the output by ~1 % mean / 10 % max.
GAMMA_RANGE = (0.25, 0.75)
BETA = (0.6, 0.25)
HOT = (0.02, 2.5, 3.5)      # fraction of encoder channels with a large gamma (drives the ReLU6 clamp)


def _probe(seed, calib_hw, in_channels):
    """The seeded calibration batch: 2 images of ``in_channels`` channels (3: the fixtures' original draw, unchanged)."""
    if in_channels == 3:
        return torch.from_numpy(np.random.Generator(np.random.PCG64(seed + 7919)).random((2, 3) + tuple(calib_hw)))
    return synthetic_input(2, calib_hw[0], calib_hw[1], seed=seed + 7919, channels=in_channels).double()


def synthetic_state_dict(widths=STOCK_WIDTHS, seed=1, calib_hw=(96, 128), skip='add', recipe='hot', in_channels=3):
    """state_dict (torch fp32 CPU tensors) with the MobileNetSkipAdd key schema
    (SURVEY.md section 8a-a2).

    BatchNorm running statistics are CALIBRATED: a seeded probe batch is pushed through the
    layers (fp64, torch CPU) and every BN's running_mean/var are set to the statistics of the
    tensor it normalises -- what training leaves behind in a real checkpoint.  That keeps the
    network well conditioned (fp16 storage noise is not chaotically amplified), so the 1e-2 fp16
    tolerance is a meaningful bound and not noise.  gamma ~ U(0.25, 0.75) with 2 % "hot" encoder
    channels at U(2.5, 3.5) that drive ~0.1 % of the activations into the ReLU6 clamp;
    beta ~ N(0.6, 0.25) leaves ~10-15 % exact zeros after each ReLU.

    ``recipe='calm'`` is the same recipe WITHOUT the hot channels: no single element's storage noise is amplified
    ~4x, so every intermediate stage can be held to the end-to-end tolerance (1e-2 in fp16) and a stage bug of a few
    percent cannot hide behind the loose stage bound the hot recipe needs (tests/test_gpu_parity.py).

    ``in_channels`` (reference ``MobileNet(..., in_channels)``, models.py:443-453) sets the stem's input channels: its
    weights are drawn as [enc[0], in_channels, 3, 3] and the probe batch is ``synthetic_input(..., channels=in_channels)``.
    With the default 3 every draw is the one above, so the existing fixtures stay bit-identical."""
    if recipe not in ('hot', 'calm'):
        raise ValueError('recipe must be "hot" or "calm"')
    hot_cfg = HOT if recipe == 'hot' else (0.0, HOT[1], HOT[2])
    key = (tuple(widths[0]), tuple(widths[1]), int(seed), tuple(calib_hw), GAMMA_RANGE, BETA, hot_cfg, skip, int(in_channels))
    if key in _CACHE:
        return {k: v.clone() for k, v in _CACHE[key].items()}
    import torch.nn.functional as F
    enc, dec = widths
    rng = np.random.Generator(np.random.PCG64(seed))
    sd = {}
    f64 = torch.float64

    def gauss(shape, fan):
        return torch.from_numpy(rng.normal(0.0, np.sqrt(2.0 / fan), shape))

    def unif(shape, fan):
        b = 1.0 / np.sqrt(fan)
        return torch.from_numpy(rng.uniform(-b, b, shape))

    def bn_act(t, c, prefix, hi, last=False):
        """draw gamma/beta, calibrate mean/var on t, store, apply BN + clamp"""
        if last:
            gamma = np.ones(c); beta = np.full(c, 3.0)          # depth-like, strictly alive head
        else:
            gamma = rng.uniform(GAMMA_RANGE[0], GAMMA_RANGE[1], c); beta = rng.normal(BETA[0], BETA[1], c)
            hot = rng.random(c) < hot_cfg[0]
            gamma = np.where(hot & (hi is not None), rng.uniform(HOT[1], HOT[2], c), gamma)
        mean = t.mean(dim=(0, 2, 3)); var = t.var(dim=(0, 2, 3), unbiased=False)
        sd[prefix + '.weight'] = torch.from_numpy(gamma).float()
        sd[prefix + '.bias'] = torch.from_numpy(beta).float()
        sd[prefix + '.running_mean'] = mean.float()
        sd[prefix + '.running_var'] = var.float()
        sd[prefix + '.num_batches_tracked'] = torch.zeros((), dtype=torch.int64)
        g, b = sd[prefix + '.weight'].to(f64), sd[prefix + '.bias'].to(f64)
        m, v = sd[prefix + '.running_mean'].to(f64), sd[prefix + '.running_var'].to(f64)
        inv = g / torch.sqrt(v + 1e-5)
        y = t * inv.view(1, -1, 1, 1) + (b - m * inv).view(1, -1, 1, 1)
        return y.clamp(0.0, hi) if hi is not None else y.clamp_min(0.0)

    def put(name, wt):
        sd[name] = wt.float().contiguous()
        return sd[name].to(f64)

    strides = (2, 1, 2, 1, 2, 1, 2, 1, 1, 1, 1, 1, 2, 1)
    x = _probe(seed, calib_hw, in_channels)
    x = bn_act(F.conv2d(x, put('conv0.0.weight', gauss((enc[0], in_channels, 3, 3), 9 * in_channels)), None, 2, 1), enc[0],
               'conv0.1', 6.0)
    keep = {}
    for i in range(1, 14):
        ci, co = enc[i - 1], enc[i]
        x = bn_act(F.conv2d(x, put('conv%d.0.weight' % i, gauss((ci, 1, 3, 3), 9)), None, strides[i], 1, 1, ci),
                   ci, 'conv%d.1' % i, 6.0)
        x = bn_act(F.conv2d(x, put('conv%d.3.weight' % i, gauss((co, ci, 1, 1), ci))), co, 'conv%d.4' % i, 6.0)
        if i in (1, 3, 5):
            keep[i] = x
    c = enc[13]
    add_after = {4: 1, 3: 3, 2: 5}
    for j, co in enumerate(dec, start=1):
        x = bn_act(F.conv2d(x, put('decode_conv%d.0.0.weight' % j, unif((c, 1, 5, 5), 25)), None, 1, 2, 1, c),
                   c, 'decode_conv%d.0.1' % j, None)
        x = bn_act(F.conv2d(x, put('decode_conv%d.1.0.weight' % j, unif((co, c, 1, 1), c))), co,
                   'decode_conv%d.1.1' % j, None)
        x = x.repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
        c = co
        if j in add_after:
            if skip == 'concat':                       # MobileNetSkipConcat (reference models.py:806-811)
                x = torch.cat((x, keep[add_after[j]]), 1)
                c = co + keep[add_after[j]].shape[1]
            else:
                x = x + keep[add_after[j]]
    bn_act(F.conv2d(x, put('decode_conv6.0.weight', unif((1, c, 1, 1), c).abs())), 1, 'decode_conv6.1', None, last=True)
    # keep the reference's key order (conv.weight first, then BN entries)
    _CACHE[key] = sd
    return {k: v.clone() for k, v in sd.items()}


SPARSE_DENSITY = 0.05          # fraction of pixels with a depth sample in a synthetic sparse-depth channel
SPARSE_RANGE = (0.5, 10.0)     # metres, the NYU Depth v2 range


def synthetic_input(n, h, w, seed=0, channels=3):
    """[n,3,h,w] fp32 in [0,1) -- the range the reference pipeline yields
    (dataloaders/transforms.py:216-224, dataloaders/nyu.py:56).

    ``channels != 3``: the input of a sparse-to-dense model, ``channels - 1`` image channels in [0, 1) and then one sparse
    depth channel in metres: zero except at a ``SPARSE_DENSITY`` fraction of the pixels, where it is U(0.5, 10).  So 4 is
    RGB-D and 1 is depth only.  ``channels=3`` is the draw above, unchanged."""
    rng = np.random.Generator(np.random.PCG64(seed))
    if channels == 3:
        return torch.from_numpy(rng.random((n, 3, h, w), dtype=np.float32))
    if channels < 1:
        raise ValueError('channels must be >= 1')
    img = rng.random((n, channels - 1, h, w), dtype=np.float32)
    hit = rng.random((n, 1, h, w)) < SPARSE_DENSITY
    depth = np.where(hit, rng.uniform(SPARSE_RANGE[0], SPARSE_RANGE[1], (n, 1, h, w)), 0.0).astype(np.float32)
    return torch.from_numpy(np.ascontiguousarray(np.concatenate([img, depth], axis=1)))


def synthetic_target(pred, seed=1):
    """Strictly positive pseudo ground truth around an oracle prediction (SURVEY.md section 8d):
    t = pred * (1 + 0.1*randn), clamped to >= 1e-3 so metrics.py's masks/logs stay finite."""
    rng = np.random.Generator(np.random.PCG64(seed))
    noise = torch.from_numpy(rng.standard_normal(tuple(pred.shape)).astype(np.float32))
    return (pred.float().cpu() * (1.0 + 0.1 * noise)).clamp_min(1e-3)


def to_mobilenet_keys(sd):
    """Rename a MobileNetSkipAdd-schema state_dict to the ``models.MobileNet(decoder='nnconv5dw')`` schema
    (``conv<i>.*`` -> ``mobilenet.<i>.*``, ``decode_conv<j>.*`` -> ``decoder.conv<j>.*``)."""
    out = {}
    for k, v in sd.items():
        if k.startswith('decode_conv'):
            j, rest = k[len('decode_conv'):].split('.', 1)
            out['decoder.conv%s.%s' % (j, rest)] = v
        else:
            i, rest = k[len('conv'):].split('.', 1)
            out['mobilenet.%s.%s' % (i, rest)] = v
    return out


def synthetic_nnconv_state_dict(kernel_size=5, seed=1, calib_hw=(96, 128), in_channels=3):
    """state_dict with the ``models.MobileNet('nnconv<k>')`` key schema (dense NNConv decoder, reference models.py:52-59,
    245-270): the encoder of ``synthetic_state_dict(STOCK_WIDTHS, seed)`` (renamed with ``to_mobilenet_keys``), then five
    dense ``conv(C, C/2, k)`` blocks and ``pointwise(32, 1)`` drawn from a separate seeded stream.

    Same recipe as the depthwise decoder: conv weights U(-b, b) with b = 1/sqrt(fan_in) (fan_in = k*k*C), BN gamma / beta
    drawn as above and running statistics CALIBRATED in fp64 on the encoder output of the same probe batch, a positive head
    with gamma = 1, beta = 3.  Measured conditioning (storage-emulated forward against the fp32 forward, seed 1): fp16
    2.5e-3 at 2x64x96 but 1.5e-2 at 1x224x224 (bf16 2.5e-2 / 1.2e-1); calibrating the decoder on a 224 x 224 probe instead
    does not change that.  The functions above are untouched, so their fixtures stay bit-identical.  ``in_channels``: the
    stem's input channels, as in ``synthetic_state_dict``."""
    import torch.nn.functional as F
    base = to_mobilenet_keys(synthetic_state_dict(STOCK_WIDTHS, seed=seed, calib_hw=calib_hw, in_channels=in_channels))
    sd = {k: v for k, v in base.items() if k.startswith('mobilenet.')}
    f64 = torch.float64

    def bn(t, prefix, hi):
        g, b = sd[prefix + '.weight'].to(f64), sd[prefix + '.bias'].to(f64)
        m, v = sd[prefix + '.running_mean'].to(f64), sd[prefix + '.running_var'].to(f64)
        inv = g / torch.sqrt(v + 1e-5)
        y = t * inv.view(1, -1, 1, 1) + (b - m * inv).view(1, -1, 1, 1)
        return y.clamp(0.0, hi) if hi is not None else y.clamp_min(0.0)

    strides = (2, 1, 2, 1, 2, 1, 2, 1, 1, 1, 1, 1, 2, 1)
    x = _probe(seed, calib_hw, in_channels)
    x = bn(F.conv2d(x, sd['mobilenet.0.0.weight'].to(f64), None, 2, 1), 'mobilenet.0.1', 6.0)
    for i in range(1, 14):
        ci = sd['mobilenet.%d.0.weight' % i].shape[0]
        x = bn(F.conv2d(x, sd['mobilenet.%d.0.weight' % i].to(f64), None, strides[i], 1, 1, ci), 'mobilenet.%d.1' % i, 6.0)
        x = bn(F.conv2d(x, sd['mobilenet.%d.3.weight' % i].to(f64)), 'mobilenet.%d.4' % i, 6.0)
    rng = np.random.Generator(np.random.PCG64(seed + 104729))
    k, c = int(kernel_size), STOCK_ENCODER[13]

    def calibrate(t, prefix, last=False):
        ch = t.shape[1]
        if last:
            gamma, beta = np.ones(ch), np.full(ch, 3.0)
        else:
            gamma, beta = rng.uniform(GAMMA_RANGE[0], GAMMA_RANGE[1], ch), rng.normal(BETA[0], BETA[1], ch)
        sd[prefix + '.weight'] = torch.from_numpy(gamma).float()
        sd[prefix + '.bias'] = torch.from_numpy(beta).float()
        sd[prefix + '.running_mean'] = t.mean(dim=(0, 2, 3)).float()
        sd[prefix + '.running_var'] = t.var(dim=(0, 2, 3), unbiased=False).float()
        sd[prefix + '.num_batches_tracked'] = torch.zeros((), dtype=torch.int64)
        return bn(t, prefix, None)

    for j, co in enumerate(STOCK_DECODER, start=1):
        b = 1.0 / np.sqrt(k * k * c)
        sd['decoder.conv%d.0.weight' % j] = torch.from_numpy(rng.uniform(-b, b, (co, c, k, k))).float().contiguous()
        x = calibrate(F.conv2d(x, sd['decoder.conv%d.0.weight' % j].to(f64), None, 1, (k - 1) // 2), 'decoder.conv%d.1' % j)
        x = x.repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
        c = co
    b = 1.0 / np.sqrt(c)
    sd['decoder.conv6.0.weight'] = torch.from_numpy(np.abs(rng.uniform(-b, b, (1, c, 1, 1)))).float().contiguous()
    calibrate(F.conv2d(x, sd['decoder.conv6.0.weight'].to(f64)), 'decoder.conv6.1', last=True)
    return sd


def synthetic_convt_state_dict(decoder, seed=1, calib_hw=(96, 128), in_channels=3):
    """state_dict with the ``models.MobileNet(decoder)`` key schema for ``decoder`` in ``deconv3/5/7/9`` and ``upconv``
    (reference models.py:77-107, 145-201): the encoder of ``synthetic_state_dict(STOCK_WIDTHS, seed)`` (renamed with
    ``to_mobilenet_keys``), then five ``convt(C, C/2, k)`` (keys ``decoder.convt<j>.{0,1}.*``) or ``upconv(C, C/2)``
    blocks (``decoder.upconv<j>.{1,2}.*``) and ``convf = pointwise(32, 1)``, drawn from a separate seeded stream.

    The recipe of ``synthetic_nnconv_state_dict``: decoder weights U(-b, b) with b = 1/sqrt(k*k*C), BN gamma / beta drawn
    as there, running statistics CALIBRATED in fp64 on the same probe batch, a positive head with gamma = 1, beta = 3.
    ``in_channels``: the stem's input channels, as in ``synthetic_state_dict``."""
    import torch.nn.functional as F
    if decoder == 'upconv':
        k, child, conv_i, bn_i = 5, 'upconv', 1, 2
    elif decoder in ('deconv3', 'deconv5', 'deconv7', 'deconv9'):
        k, child, conv_i, bn_i = int(decoder[6]), 'convt', 0, 1
    else:
        raise ValueError('no synthetic recipe for decoder %r' % decoder)
    base = to_mobilenet_keys(synthetic_state_dict(STOCK_WIDTHS, seed=seed, calib_hw=calib_hw, in_channels=in_channels))
    sd = {key: v for key, v in base.items() if key.startswith('mobilenet.')}
    f64 = torch.float64

    def bn(t, prefix, hi):
        g, b = sd[prefix + '.weight'].to(f64), sd[prefix + '.bias'].to(f64)
        m, v = sd[prefix + '.running_mean'].to(f64), sd[prefix + '.running_var'].to(f64)
        inv = g / torch.sqrt(v + 1e-5)
        y = t * inv.view(1, -1, 1, 1) + (b - m * inv).view(1, -1, 1, 1)
        return y.clamp(0.0, hi) if hi is not None else y.clamp_min(0.0)

    strides = (2, 1, 2, 1, 2, 1, 2, 1, 1, 1, 1, 1, 2, 1)
    x = _probe(seed, calib_hw, in_channels)
    x = bn(F.conv2d(x, sd['mobilenet.0.0.weight'].to(f64), None, 2, 1), 'mobilenet.0.1', 6.0)
    for i in range(1, 14):
        ci = sd['mobilenet.%d.0.weight' % i].shape[0]
        x = bn(F.conv2d(x, sd['mobilenet.%d.0.weight' % i].to(f64), None, strides[i], 1, 1, ci), 'mobilenet.%d.1' % i, 6.0)
        x = bn(F.conv2d(x, sd['mobilenet.%d.3.weight' % i].to(f64)), 'mobilenet.%d.4' % i, 6.0)
    rng = np.random.Generator(np.random.PCG64(seed + 104729))
    c = STOCK_ENCODER[13]

    def calibrate(t, prefix, last=False):
        ch = t.shape[1]
        if last:
            gamma, beta = np.ones(ch), np.full(ch, 3.0)
        else:
            gamma, beta = rng.uniform(GAMMA_RANGE[0], GAMMA_RANGE[1], ch), rng.normal(BETA[0], BETA[1], ch)
        sd[prefix + '.weight'] = torch.from_numpy(gamma).float()
        sd[prefix + '.bias'] = torch.from_numpy(beta).float()
        sd[prefix + '.running_mean'] = t.mean(dim=(0, 2, 3)).float()
        sd[prefix + '.running_var'] = t.var(dim=(0, 2, 3), unbiased=False).float()
        sd[prefix + '.num_batches_tracked'] = torch.zeros((), dtype=torch.int64)
        return bn(t, prefix, None)

    for j, co in enumerate(STOCK_DECODER, start=1):
        b = 1.0 / np.sqrt(k * k * c)
        key = 'decoder.%s%d.%d.weight' % (child, j, conv_i)
        if child == 'convt':
            sd[key] = torch.from_numpy(rng.uniform(-b, b, (c, co, k, k))).float().contiguous()
            y = F.conv_transpose2d(x, sd[key].to(f64), None, 2, (k - 1) // 2, 1)
        else:
            sd[key] = torch.from_numpy(rng.uniform(-b, b, (co, c, k, k))).float().contiguous()
            u = x.new_zeros(x.shape[0], c, x.shape[2], 2, x.shape[3], 2)
            u[:, :, :, 0, :, 0] = x
            y = F.conv2d(u.view(x.shape[0], c, 2 * x.shape[2], 2 * x.shape[3]), sd[key].to(f64), None, 1, 2)
        x = calibrate(y, 'decoder.%s%d.%d' % (child, j, bn_i))
        c = co
    b = 1.0 / np.sqrt(c)
    sd['decoder.convf.0.weight'] = torch.from_numpy(np.abs(rng.uniform(-b, b, (1, c, 1, 1)))).float().contiguous()
    calibrate(F.conv2d(x, sd['decoder.convf.0.weight'].to(f64)), 'decoder.convf.1', last=True)
    return sd
