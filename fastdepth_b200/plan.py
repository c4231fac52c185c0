"""Host-side planning: read a MobileNetSkipAdd-shaped module, fold BatchNorm, describe the
stages and hand everything to the C-ABI.

The module is only *read* here (conv weights, BN statistics, strides): attribute access is
limited to ``.weight/.stride/.kernel_size/.groups`` of convs and
``.weight/.bias/.running_mean/.running_var/.eps`` of BNs so that modules unpickled from old
PyTorch versions (missing newer attributes) still work (SURVEY.md section 5, checkpoint row).
"""
import ctypes

import numpy as np
import torch
import torch.nn as nn

from . import _lib
from ._lib import StageDesc

DTYPE_CODE = {torch.float32: _lib.FD_F32, torch.float16: _lib.FD_F16, torch.bfloat16: _lib.FD_BF16}
N_METRICS = 11
METRIC_NAMES = ('irmse', 'imae', 'mse', 'rmse', 'mae', 'absrel', 'lg10', 'delta1', 'delta2', 'delta3')

# encoder block i -> skip consumer: decode stage j adds the output of encoder block SKIP[j]
# (reference models.py:714-719, 724-729)
SKIP_FOR_DECODE = {2: 5, 3: 3, 4: 1}


def fold_bn(bn):
    """Eval-mode BatchNorm2d as y = x*scale + bias, folded in fp32 (exact to ~4e-6 rel).
    reference: nn.BatchNorm2d in conv_bn/conv_dw/depthwise/pointwise, eps 1e-5."""
    g = bn.weight.detach().float().cpu()
    b = bn.bias.detach().float().cpu()
    m = bn.running_mean.detach().float().cpu()
    v = bn.running_var.detach().float().cpu()
    scale = g / torch.sqrt(v + float(bn.eps))
    bias = b - m * scale
    return scale.contiguous().numpy(), bias.contiguous().numpy()


def _act_of(m):
    if isinstance(m, nn.ReLU6):
        return _lib.FD_ACT_RELU6
    if isinstance(m, nn.ReLU):
        return _lib.FD_ACT_RELU
    raise RuntimeError('unsupported activation %r on the hot path' % type(m).__name__)


def _w(conv):
    return np.ascontiguousarray(conv.weight.detach().float().cpu().numpy())


def _sq(v):
    return int(v[0]) if isinstance(v, (tuple, list)) else int(v)


def _blocks_of(module):
    """(encoder blocks[14], decoder blocks[5], head, skips?) for the module shapes on the hot path:
    ``MobileNetSkipAdd`` (children conv0..13, decode_conv1..6; reference models.py:674-698) and
    ``MobileNet`` with an NNConv decoder, depthwise or dense (children mobilenet[0..13], decoder.conv1..6; reference
    models.py:229-270, 441-455)."""
    if hasattr(module, 'conv0') and hasattr(module, 'decode_conv6'):
        enc = [getattr(module, 'conv%d' % i) for i in range(14)]
        dec = [getattr(module, 'decode_conv%d' % j) for j in range(1, 6)]
        names = ['conv%d' % i for i in range(14)] + ['decode_conv%d' % j for j in range(1, 7)]
        # MobileNetSkipConcat (reference models.py:734-814) has the same children; its decoder blocks 3..5 take the
        # concatenation [upsampled, skip] -- recognisable by class name (pickles) or by the widened depthwise convs
        concat = type(module).__name__ == 'MobileNetSkipConcat' or \
            dec[2][0][0].weight.shape[0] != dec[1][1][0].weight.shape[0]
        return enc, dec, module.decode_conv6, ('concat' if concat else True), names
    if hasattr(module, 'mobilenet') and hasattr(module, 'decoder'):
        enc = [module.mobilenet[i] for i in range(14)]
        for child in ('convt', 'upconv'):          # DeConv / UpConv decoders (reference models.py:145-201)
            if hasattr(module.decoder, child + '1'):
                dec = [getattr(module.decoder, '%s%d' % (child, j)) for j in range(1, 6)]
                names = ['mobilenet.%d' % i for i in range(14)] + ['decoder.%s%d' % (child, j) for j in range(1, 6)]
                return enc, dec, module.decoder.convf, False, names + ['decoder.convf']
        dec = [getattr(module.decoder, 'conv%d' % j) for j in range(1, 6)]
        names = ['mobilenet.%d' % i for i in range(14)] + ['decoder.conv%d' % j for j in range(1, 7)]
        return enc, dec, module.decoder.conv6, False, names
    raise RuntimeError('unsupported module for the fastdepth_b200 hot path: %s' % type(module).__name__)


def _is_dense_block(b):
    """conv(C, C', k) of the dense NNConv decoder (reference models.py:52-59): Conv2d(groups 1, stride 1, k in {3, 5}),
    BatchNorm2d, ReLU."""
    return (isinstance(b, nn.Sequential) and len(b) == 3 and isinstance(b[0], nn.Conv2d) and b[0].groups == 1 and
            _sq(b[0].kernel_size) in (3, 5) and _sq(b[0].stride) == 1 and isinstance(b[1], nn.BatchNorm2d))


def _convt_kind(b):
    """FD_STAGE_DECONV for convt(C, C', k) (ConvTranspose2d(k in 3/5/7/9, stride 2, padding (k-1)/2, output_padding 1),
    BN, ReLU; reference models.py:77-87), FD_STAGE_UPCONV for upconv(C, C') (Unpool(2), Conv2d(5, 1, 2), BN, ReLU;
    l.101-107), else None."""
    if not isinstance(b, nn.Sequential):
        return None
    if len(b) == 3 and isinstance(b[0], nn.ConvTranspose2d) and isinstance(b[1], nn.BatchNorm2d):
        c, k = b[0], _sq(b[0].kernel_size)
        ok = (k in (3, 5, 7, 9) and c.groups == 1 and _sq(c.stride) == 2 and _sq(c.padding) == (k - 1) // 2 and
              _sq(c.output_padding) == 1 and _sq(c.dilation) == 1 and c.bias is None)
        return _lib.FD_STAGE_DECONV if ok else None
    if len(b) == 4 and type(b[0]).__name__ == 'Unpool' and isinstance(b[1], nn.Conv2d) and isinstance(b[2], nn.BatchNorm2d):
        c = b[1]
        ok = (getattr(b[0], 'stride', None) == 2 and _sq(c.kernel_size) == 5 and c.groups == 1 and _sq(c.stride) == 1 and
              _sq(c.padding) == 2 and _sq(c.dilation) == 1 and c.bias is None)
        return _lib.FD_STAGE_UPCONV if ok else None
    return None


def dense_decoder(module):
    """True if the module's decoder is dense: the NNConv decoder (``MobileNet('nnconv5')`` / ``('nnconv3')``) or the
    DeConv / UpConv decoder (``MobileNet('deconv<k>')`` / ``('upconv')``)."""
    try:
        _, dec, _, _, _ = _blocks_of(module)
        return all(_is_dense_block(b) for b in dec) or all(_convt_kind(b) is not None for b in dec)
    except Exception:
        return False


def supports(module):
    """True if ``describe`` can express the module: depthwise-separable decoder blocks of two Sequentials, dense
    k x k conv blocks (k in {3, 5}) of the NNConv decoder, or the transposed-conv / unpool blocks of DeConv / UpConv."""
    try:
        enc, dec, head, _, _ = _blocks_of(module)
        return all(isinstance(b, nn.Sequential) and len(b) == 2 and isinstance(b[0], nn.Sequential) and
                   b[0][0].groups == b[0][0].in_channels for b in dec) or dense_decoder(module)
    except Exception:
        return False


def describe(module):
    """Walk the 14 encoder blocks, 5 decoder blocks and the head and return (stage descs, per-stage weight
    tuples, stage names).

    Mirrors the dispatch of reference models.py:706-732 (SkipAdd: skips saved after encoder blocks 1/3/5 and added
    after decoder stages 4/3/2) and models.py:253-270, 457-460 (MobileNet + NNConv: no skips; a dense decoder block
    becomes one CONV stage with the weight tuple ``(None, None, None, w.reshape(c_out, -1), scale, bias)``; a DeConv /
    UpConv block becomes one DECONV / UPCONV stage with the module's own weight, flattened behind its first axis)."""
    enc, dec, hd, with_skips, names = _blocks_of(module)
    descs, weights = [], []
    conv0 = enc[0]
    c, bn, act = conv0[0], conv0[1], conv0[2]
    descs.append(dict(kind=_lib.FD_STAGE_STEM, c_in=c.weight.shape[1], c_out=c.weight.shape[0],
                      ksize=_sq(c.kernel_size), stride=_sq(c.stride), act=_act_of(act), upsample=0, skip_src=-1))
    s, b = fold_bn(bn)
    weights.append((None, None, None, _w(c), s, b))
    stage_of_encoder = {0: 0}
    for i in range(1, 14):
        blk = enc[i]
        dw, bn1, a1, pw, bn2, a2 = blk[0], blk[1], blk[2], blk[3], blk[4], blk[5]
        if _act_of(a1) != _act_of(a2):
            raise RuntimeError('encoder block %d: mixed activations are not supported' % i)
        descs.append(dict(kind=_lib.FD_STAGE_DWPW, c_in=dw.weight.shape[0], c_out=pw.weight.shape[0],
                          ksize=_sq(dw.kernel_size), stride=_sq(dw.stride), act=_act_of(a1), upsample=0, skip_src=-1))
        s1, b1 = fold_bn(bn1)
        s2, b2 = fold_bn(bn2)
        weights.append((_w(dw).reshape(dw.weight.shape[0], -1), s1, b1,
                        _w(pw).reshape(pw.weight.shape[0], pw.weight.shape[1]), s2, b2))
        stage_of_encoder[i] = len(descs) - 1
    for j in range(1, 6):
        blk = dec[j - 1]
        kind = _convt_kind(blk)
        if kind is not None:
            # convt(): ConvTranspose2d weights [c_in][c_out][k][k]; upconv(): Unpool, then Conv2d weights [c_out][c_in][5][5]
            c, bn, a = (blk[0], blk[1], blk[2]) if kind == _lib.FD_STAGE_DECONV else (blk[1], blk[2], blk[3])
            c_in, c_out = (c.weight.shape[0], c.weight.shape[1]) if kind == _lib.FD_STAGE_DECONV else \
                (c.weight.shape[1], c.weight.shape[0])
            descs.append(dict(kind=kind, c_in=c_in, c_out=c_out, ksize=_sq(c.kernel_size), stride=2, act=_act_of(a),
                              upsample=0, skip_src=-1))
            s, b = fold_bn(bn)
            weights.append((None, None, None, _w(c).reshape(c.weight.shape[0], -1), s, b))
            continue
        if _is_dense_block(blk):
            # dense kxk conv + BN + ReLU, then the nearest x2 upsample (reference models.py:52-59, 261-270)
            c, bn, a = blk[0], blk[1], blk[2]
            descs.append(dict(kind=_lib.FD_STAGE_CONV, c_in=c.weight.shape[1], c_out=c.weight.shape[0],
                              ksize=_sq(c.kernel_size), stride=1, act=_act_of(a), upsample=1, skip_src=-1))
            s, b = fold_bn(bn)
            weights.append((None, None, None, _w(c).reshape(c.weight.shape[0], -1), s, b))
            continue
        (dw, bn1, a1), (pw, bn2, a2) = (blk[0][0], blk[0][1], blk[0][2]), (blk[1][0], blk[1][1], blk[1][2])
        if _act_of(a1) != _act_of(a2):
            raise RuntimeError('decoder block %d: mixed activations are not supported' % j)
        skip = stage_of_encoder[SKIP_FOR_DECODE[j]] if (with_skips and j in SKIP_FOR_DECODE) else -1
        descs.append(dict(kind=_lib.FD_STAGE_DWPW, c_in=dw.weight.shape[0], c_out=pw.weight.shape[0],
                          ksize=_sq(dw.kernel_size), stride=1, act=_act_of(a1), upsample=1, skip_src=skip,
                          skip_mode=1 if (with_skips == 'concat' and skip >= 0) else 0))
        s1, b1 = fold_bn(bn1)
        s2, b2 = fold_bn(bn2)
        weights.append((_w(dw).reshape(dw.weight.shape[0], -1), s1, b1,
                        _w(pw).reshape(pw.weight.shape[0], pw.weight.shape[1]), s2, b2))
    c, bn, act = hd[0], hd[1], hd[2]
    descs.append(dict(kind=_lib.FD_STAGE_HEAD, c_in=c.weight.shape[1], c_out=1, ksize=1, stride=1,
                      act=_act_of(act), upsample=0, skip_src=-1))
    s, b = fold_bn(bn)
    weights.append((None, None, None, _w(c).reshape(1, -1), s, b))
    return descs, weights, names


def _fp(a):
    if a is None:
        return None
    assert a.dtype == np.float32 and a.flags['C_CONTIGUOUS']
    return a.ctypes.data_as(ctypes.c_void_p)


class Plan:
    """Owns one ``fd_plan`` built for (N, H, W, dtype, device); ``forward`` runs any (n, h, w) with h, w multiples of 32 and
    n*h*w <= N*H*W.  Thin: every method is one C-ABI call."""

    def __init__(self, descs, weights, names, n, h, w, dtype, device_index):
        self.lib = _lib.load()
        self.n, self.h, self.w, self.dtype = n, h, w, dtype
        self.device_index = device_index
        self.names = list(names)
        arr = (StageDesc * len(descs))(*[StageDesc(**d) for d in descs])
        handle = ctypes.c_void_p()
        _lib.check(self.lib.fd_plan_create(arr, len(descs), n, h, w, DTYPE_CODE[dtype], device_index,
                                           ctypes.byref(handle)))
        self.handle = handle
        self.set_weights(weights)

    @classmethod
    def from_module(cls, module, n, h, w, dtype, device_index):
        descs, weights, names = describe(module)
        return cls(descs, weights, names, n, h, w, dtype, device_index)

    def set_weights(self, weights):
        for i, wt in enumerate(weights):
            keep = [np.ascontiguousarray(a, dtype=np.float32) if a is not None else None for a in wt]
            _lib.check(self.lib.fd_plan_set_stage_weights(self.handle, i, *[_fp(a) for a in keep]))

    def set_option(self, name, value):
        _lib.check(self.lib.fd_plan_set_option(self.handle, name.encode(), int(value)))

    def get_option(self, name):
        v = ctypes.c_int()
        _lib.check(self.lib.fd_plan_get_option(self.handle, name.encode(), ctypes.byref(v)))
        return v.value

    def forward(self, x, y, stream_ptr, n=None):
        """Forward of the first ``n`` images (default ``x.shape[0]``) of ``x`` at its own resolution, through
        ``fd_forward_shape``: any shape whose pixels n*h*w fit the plan's n*h*w runs on the plan's buffers."""
        n = x.shape[0] if n is None else int(n)
        _lib.check(self.lib.fd_forward_shape(self.handle, n, x.shape[2], x.shape[3], x.data_ptr(), y.data_ptr(),
                                             stream_ptr))

    def forward_host(self, x_host, y_host, stream_ptr):
        _lib.check(self.lib.fd_forward_host(self.handle, x_host.data_ptr(), y_host.data_ptr(), stream_ptr))

    def pipeline_submit(self, x_host, y_host):
        """Asynchronous H2D -> forward -> D2H of one pinned host batch; returns a ticket (fd_pipeline_submit)."""
        t = ctypes.c_uint64()
        _lib.check(self.lib.fd_pipeline_submit(self.handle, x_host.data_ptr(), y_host.data_ptr(), ctypes.byref(t)))
        return t.value

    def pipeline_wait(self, ticket):
        _lib.check(self.lib.fd_pipeline_wait(self.handle, ticket))

    def launches_per_forward(self):
        v = ctypes.c_int()
        _lib.check(self.lib.fd_plan_launches_per_forward(self.handle, ctypes.byref(v)))
        return v.value

    def workspace_bytes(self):
        v = ctypes.c_size_t()
        _lib.check(self.lib.fd_plan_workspace_bytes(self.handle, ctypes.byref(v)))
        return v.value

    def steps(self):
        n = ctypes.c_int()
        _lib.check(self.lib.fd_plan_step_count(self.handle, ctypes.byref(n)))
        out = []
        for i in range(n.value):
            st, ab, mc = ctypes.c_int(), ctypes.c_double(), ctypes.c_double()
            buf = ctypes.create_string_buffer(200)
            _lib.check(self.lib.fd_plan_step_info(self.handle, i, ctypes.byref(st), ctypes.byref(ab), ctypes.byref(mc),
                                                  buf, 200))
            dwm, dnm = ctypes.c_double(), ctypes.c_double()
            _lib.check(self.lib.fd_plan_step_macs(self.handle, i, ctypes.byref(dwm), ctypes.byref(dnm)))
            kname = buf.value.decode()
            sname = self.names[st.value]
            if 'chain_tc' in kname and '{stages ' in kname:            # one kernel for a run of stages: name the run
                a, b = kname.split('{stages ')[1].rstrip('}').split('-')
                sname = '%s..%s' % (self.names[int(a)], self.names[int(b)])
            out.append(dict(step=i, stage=st.value, stage_name=sname, kernel=kname,
                            alg_bytes=ab.value, macs=mc.value, dw_macs=dwm.value, dense_macs=dnm.value))
        return out

    def time_steps(self, x, y, stream_ptr, warmup=3, iters=20, flush_l2=True):
        steps = self.steps()
        ms = (ctypes.c_float * len(steps))()
        _lib.check(self.lib.fd_plan_time_steps(self.handle, x.data_ptr(), y.data_ptr(), stream_ptr, warmup, iters,
                                               1 if flush_l2 else 0, ms))
        for s, t in zip(steps, ms):
            s['ms'] = float(t)
        return steps

    def trace_stage(self, stage, y, stream_ptr):
        """Debug timeline of one fused block kernel (CTA 0): dict row-name -> list of SM clock stamps."""
        import numpy as np
        buf = (ctypes.c_uint64 * 3072)()
        rows, cols = ctypes.c_int(), ctypes.c_int()
        _lib.check(self.lib.fd_plan_trace_stage(self.handle, stage, y.data_ptr(), stream_ptr, buf, 3072,
                                                ctypes.byref(rows), ctypes.byref(cols)))
        a = np.frombuffer(buf, dtype=np.uint64).reshape(rows.value, cols.value).astype(np.int64)
        in_chain = False
        for st in self.steps():
            if 'chain_tc' in st['kernel'] and '{stages ' in st['kernel']:
                lo, hi = st['kernel'].split('{stages ')[1].rstrip('}').split('-')
                in_chain = in_chain or int(lo) <= stage <= int(hi)
        if in_chain:
            cnames = ('layer_start', 'dw_first_kb_computed', 'dw_done_grp0', 'pointwise_done', 'epilogue_done', 'local_barrier',
                      'halo_received', 'mma_first_a_full', 'mma_last_pass_done', 'dw_done_grp1', 'tma_first_b_issue', 'unused11')
            return {n: a[i][a[i] > 0] for i, n in enumerate(cnames)}
        names = ('tma_issue', 'dw_start', 'dw_math_done', 'a_published', 'mma_ready', 'mma_issued', 'unused6', 'epi_done',
                 'unused8', 'epi_staged', 'epi_barrier', 'epi_store_issued')
        return {n: a[i][a[i] > 0] for i, n in enumerate(names)}

    def stage_tensor(self, stage, which=0):  # noqa: C901
        """NHWC view (torch tensor aliasing plan memory) of a stage buffer, for parity tests."""
        ptr = ctypes.c_void_p()
        n, h, w, c, cs = (ctypes.c_int() for _ in range(5))
        _lib.check(self.lib.fd_stage_buffer(self.handle, stage, which, ctypes.byref(ptr), ctypes.byref(n),
                                            ctypes.byref(h), ctypes.byref(w), ctypes.byref(c), ctypes.byref(cs)))
        # the buffer may be a channel slice of a wider (concat) tensor: pixel pitch cs >= c
        numel = (n.value * h.value * w.value - 1) * cs.value + c.value
        flat = _alias_device_memory(ptr.value, (numel,), numel, self.dtype, self.device_index)
        return flat.as_strided((n.value, h.value, w.value, c.value),
                               (h.value * w.value * cs.value, w.value * cs.value, cs.value, 1))

    def close(self):
        if getattr(self, 'handle', None):
            self.lib.fd_plan_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _CudaArrayView:
    """Minimal __cuda_array_interface__ wrapper so torch can alias plan-owned memory."""

    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {'data': (ptr, False), 'shape': shape, 'typestr': typestr, 'version': 3,
                                         'strides': None}


def _alias_device_memory(ptr, shape, numel, dtype, device_index):
    if dtype == torch.float32:
        with torch.cuda.device(device_index):
            return torch.as_tensor(_CudaArrayView(ptr, (numel,), '<f4'), device='cuda:%d' % device_index).view(shape)
    with torch.cuda.device(device_index):
        raw = torch.as_tensor(_CudaArrayView(ptr, (numel,), '<i2'), device='cuda:%d' % device_index)
    return raw.view(dtype).view(shape)


def metrics_accumulate(pred, target, sums):
    """fd_metrics_accumulate: per-image metrics of ``pred`` [n,1,h,w] vs ``target`` added into the
    11-double device vector ``sums`` (reference metrics.py:31-55 per image + AverageMeter sums)."""
    lib = _lib.load()
    assert pred.is_cuda and target.is_cuda and sums.is_cuda and sums.dtype == torch.float64 and sums.numel() == N_METRICS
    pred = pred.contiguous()
    target = target.contiguous().float()
    n = pred.shape[0]
    hw = pred[0].numel()
    stream = torch.cuda.current_stream(pred.device).cuda_stream
    _lib.check(lib.fd_metrics_accumulate(pred.data_ptr(), target.data_ptr(), DTYPE_CODE[pred.dtype], n, hw,
                                         sums.data_ptr(), pred.device.index, stream))
