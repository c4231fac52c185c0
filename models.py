"""FastDepth model surface, H100-native.

This module keeps the *names* the reference harness and its pickled
checkpoints resolve (``models.MobileNetSkipAdd``, ``models.MobileNet``,
``models.choose_decoder``, ``models.weights_init`` ... -- reference
models.py:36-75, 224-270, 335-360, 420-460, 654-732) while the forward of the
hot path, ``MobileNetSkipAdd.forward`` (reference models.py:706-732), is
executed by hand-written sm_90a kernels behind the C-ABI in
``include/fastdepth_b200.h``.

What is here and what is not (SURVEY.md section 2 / section 8):

* ``MobileNetSkipAdd``  -- the accelerated class. Same ctor signature, same
  child names (``conv0..conv13``, ``decode_conv1..decode_conv6``), same
  ``state_dict`` schema.  ``forward`` on a CUDA tensor builds (lazily, so it
  survives ``__init__``-less unpickling, reference main.py:49-57) a
  ``fastdepth_b200`` plan and makes one C-ABI call.  There is NO CPU fallback
  and NO PyTorch-eager fallback: a missing extension or a CPU tensor raises.
* ``MobileNet`` + ``NNConv``  -- BASELINE config 1 plumbing
  ("MobileNet-NNConv5", dense or depthwise decoder, no skips).  On CPU it is plain
  PyTorch exactly like the reference.  A CUDA tensor through the depthwise decoder
  ("MobileNet-NNConv5(depthwise)", SURVEY.md section 8f row 2) takes the same fused
  kernels as MobileNetSkipAdd; an fp16 / bf16 CUDA tensor through the dense decoder
  ("MobileNet-NNConv5") runs the encoder on those kernels and every dense 5x5 decoder
  conv on the implicit-GEMM wgmma kernel (fd_conv_tc.cu).  The dense decoder in fp32
  stays on stock PyTorch: the project's fp32 path is SIMT, while cuDNN may run fp32
  convolutions on TF32 tensor cores (tools/bench_nnconv5.py measures both).
* ``MobileNet`` + ``DeConv`` / ``UpConv``  -- the decoder ablation of the paper
  ("MobileNet-DeConv{3,5,7,9}", "MobileNet-UpConv"): plain PyTorch on the CPU; an fp16 / bf16
  CUDA tensor runs every transposed conv (or unpool + 5x5 conv) as four stride-1 phase convs
  on the same wgmma kernel (DESIGN.md section 3.6b); fp32 stays on stock PyTorch.
* every other decoder/encoder family of the reference (DeConv with depthwise convs, UpProj,
  BLConv, ShuffleConv, ResNet*) is out of scope of this tier; ``choose_decoder``
  names them in its error.
* ``MobileNetSkipConcat``  -- SURVEY.md section 8f row 1: the concat-skip variant
  (reference models.py:734-814) on the same fused kernels; the concatenation is
  a channel-slice write into one wide NHWC buffer, never a copy.
"""
import math
import os
from collections import OrderedDict

import torch
import torch.nn as nn
import torch.nn.functional as F

import imagenet.mobilenet

_IMAGENET_CKPT = os.path.join('imagenet', 'results', 'imagenet.arch=mobilenet.lr=0.1.bs=256',
                              'model_best.pth.tar')
_SKIP_AFTER = {1: 'x1', 3: 'x2', 5: 'x3'}          # encoder block -> saved skip (ref models.py:714-719)
_ADD_AFTER = {4: 'x1', 3: 'x2', 2: 'x3'}           # decoder stage -> skip added (ref models.py:724-729)


# --------------------------------------------------------------------------------------
# initialisation + building blocks (reference models.py:36-75)
# --------------------------------------------------------------------------------------
def weights_init(m):
    """Gaussian init for conv / transposed conv, unit BN (reference models.py:36-50).

    Like the reference this dispatches on the *exact* module handed in, so calling it
    on an ``nn.Sequential`` is a no-op (SURVEY.md section 2, ``weights_init`` quirk)."""
    if isinstance(m, (nn.Conv2d, nn.ConvTranspose2d)):
        fan = m.out_channels if isinstance(m, nn.Conv2d) else m.in_channels
        std = math.sqrt(2.0 / (m.kernel_size[0] * m.kernel_size[1] * fan))
        with torch.no_grad():
            m.weight.normal_(0.0, std)
            if m.bias is not None:
                m.bias.zero_()
    elif isinstance(m, nn.BatchNorm2d):
        with torch.no_grad():
            m.weight.fill_(1.0)
            m.bias.zero_()


def _same_pad(kernel_size):
    pad = (kernel_size - 1) // 2
    if 2 * pad != kernel_size - 1:
        raise AssertionError("parameters incorrect. kernel={}, padding={}".format(kernel_size, pad))
    return pad


def _cbr(c_in, c_out, k, groups=1):
    return nn.Sequential(
        nn.Conv2d(c_in, c_out, k, stride=1, padding=_same_pad(k), bias=False, groups=groups),
        nn.BatchNorm2d(c_out),
        nn.ReLU(inplace=True))


class Unpool(nn.Module):
    """x2 unpooling with zero padding (reference models.py:18-34): every input pixel lands at the top-left corner of
    its 2x2 output block, the other three are zero.  ``mask`` ([1, 0; 0, 0]) is a plain attribute, not a buffer, as in the
    reference, so that whole-module pickles and state_dicts keep their keys."""

    def __init__(self, stride=2):
        super().__init__()
        self.stride = stride
        self.mask = torch.zeros(1, 1, stride, stride)
        self.mask[:, :, 0, 0] = 1

    def forward(self, x):
        assert x.dim() == 4
        n, c, h, w = x.shape
        s = self.stride
        out = x.new_zeros(n, c, h, s, w, s)
        out[:, :, :, 0, :, 0] = x
        return out.view(n, c, h * s, w * s)


def convt(in_channels, out_channels, kernel_size):
    """ConvTranspose2d(k, stride 2, padding (k-1)/2, output_padding k % 2) + BN + ReLU: exactly x2 (reference
    models.py:77-87)."""
    pad, out_pad = (kernel_size - 1) // 2, kernel_size % 2
    if kernel_size + out_pad - 2 * pad != 2:
        raise AssertionError("deconv parameters incorrect")
    return nn.Sequential(
        nn.ConvTranspose2d(in_channels, out_channels, kernel_size, 2, pad, out_pad, bias=False),
        nn.BatchNorm2d(out_channels),
        nn.ReLU(inplace=True))


def upconv(in_channels, out_channels):
    """Unpool(2) -> 5x5 conv -> BN -> ReLU (reference models.py:101-107)."""
    return nn.Sequential(
        Unpool(2),
        nn.Conv2d(in_channels, out_channels, kernel_size=5, stride=1, padding=2, bias=False),
        nn.BatchNorm2d(out_channels),
        nn.ReLU())


def conv(in_channels, out_channels, kernel_size):
    """Dense kxk conv + BN + ReLU (reference models.py:52-59)."""
    return _cbr(in_channels, out_channels, kernel_size)


def depthwise(in_channels, kernel_size):
    """Depthwise kxk conv + BN + ReLU (reference models.py:61-68)."""
    return _cbr(in_channels, in_channels, kernel_size, groups=in_channels)


def pointwise(in_channels, out_channels):
    """1x1 conv + BN + ReLU (reference models.py:70-75)."""
    return _cbr(in_channels, out_channels, 1)


# --------------------------------------------------------------------------------------
# config-1 plumbing: MobileNet + NNConv decoder, plain PyTorch (reference models.py:224-270, 420-460)
# --------------------------------------------------------------------------------------
class NNConv(nn.Module):
    """5 x (conv block -> nearest x2) + pointwise(32,1)  (reference models.py:224-270)."""
    CHANNELS = (1024, 512, 256, 128, 64, 32)

    def __init__(self, kernel_size, dw):
        super().__init__()
        ch = self.CHANNELS
        for i in range(5):
            if dw:
                blk = nn.Sequential(depthwise(ch[i], kernel_size), pointwise(ch[i], ch[i + 1]))
            else:
                blk = conv(ch[i], ch[i + 1], kernel_size)
            setattr(self, 'conv%d' % (i + 1), blk)
        self.conv6 = pointwise(ch[5], 1)

    def forward(self, x):
        for i in range(1, 6):
            x = getattr(self, 'conv%d' % i)(x)
            x = F.interpolate(x, scale_factor=2, mode='nearest')
        return self.conv6(x)


_DECODER_CHANNELS = (1024, 512, 256, 128, 64, 32)


class DeConv(nn.Module):
    """5 x convt(C, C/2, k) + pointwise(32, 1) (reference models.py:145-180), children ``convt1..5`` and ``convf``.  The
    depthwise variant (``deconv<k>dw``) is not built here."""

    def __init__(self, kernel_size, dw):
        super().__init__()
        if dw:
            raise NotImplementedError("decoder 'deconv%ddw' is out of scope of the H100 hot-path build; see DESIGN.md"
                                      % kernel_size)
        ch = _DECODER_CHANNELS
        for i in range(5):
            setattr(self, 'convt%d' % (i + 1), convt(ch[i], ch[i + 1], kernel_size))
        self.convf = pointwise(ch[5], 1)

    def forward(self, x):
        for i in range(1, 6):
            x = getattr(self, 'convt%d' % i)(x)
        return self.convf(x)


class UpConv(nn.Module):
    """5 x upconv(C, C/2) + pointwise(32, 1) (reference models.py:183-201), children ``upconv1..5`` and ``convf``."""

    def __init__(self):
        super().__init__()
        ch = _DECODER_CHANNELS
        for i in range(5):
            setattr(self, 'upconv%d' % (i + 1), upconv(ch[i], ch[i + 1]))
        self.convf = pointwise(ch[5], 1)

    def forward(self, x):
        for i in range(1, 6):
            x = getattr(self, 'upconv%d' % i)(x)
        return self.convf(x)


_OUT_OF_SCOPE_DECODERS = ('upproj', 'shuffle', 'blconv')


def choose_decoder(decoder):
    """String -> decoder factory (reference models.py:335-360).

    ``nnconv<k>`` / ``nnconv<k>dw``, ``deconv<k>`` (k in 3, 5, 7, 9) and ``upconv`` are supported; ``deconv<k>dw`` and the
    other ablation decoders of the paper are outside this build's scope (SURVEY.md section 2) and raise
    NotImplementedError."""
    use_dw = 'dw' in decoder
    if decoder[:6] == 'nnconv':
        assert len(decoder) == 7 or (len(decoder) == 9 and use_dw)
        model = NNConv(int(decoder[6]), use_dw)
    elif decoder[:6] == 'deconv':
        assert len(decoder) == 7 or (len(decoder) == 9 and use_dw)
        model = DeConv(int(decoder[6]), use_dw)
    elif decoder == 'upconv':
        model = UpConv()
    elif any(decoder.startswith(p) for p in _OUT_OF_SCOPE_DECODERS):
        raise NotImplementedError(
            "decoder '%s' is out of scope of the H100 hot-path build (nnconv*, deconv3/5/7/9, upconv); see DESIGN.md" % decoder)
    else:
        assert False, "invalid option for decoder: {}".format(decoder)
    model.apply(weights_init)
    return model


def _load_imagenet_encoder(mobilenet):
    """reference models.py:660-670: DataParallel checkpoint, strip the ``module.`` prefix."""
    checkpoint = torch.load(_IMAGENET_CKPT, weights_only=False)
    stripped = OrderedDict((k[7:], v) for k, v in checkpoint['state_dict'].items())
    mobilenet.load_state_dict(stripped)


class MobileNet(nn.Module):
    """MobileNet encoder + ``choose_decoder`` decoder, no skips (reference models.py:420-460)."""

    def __init__(self, decoder, output_size, in_channels=3, pretrained=True):
        super().__init__()
        self.output_size = output_size
        backbone = imagenet.mobilenet.MobileNet()
        if pretrained:
            _load_imagenet_encoder(backbone)
        else:
            backbone.apply(weights_init)
        blocks = [backbone.model[i] for i in range(14)]
        if in_channels != 3:
            blocks[0] = imagenet.mobilenet.stem_block(in_channels, 32, 2)
        self.mobilenet = nn.Sequential(*blocks)
        self.decoder = choose_decoder(decoder)

    def __getstate__(self):
        state = self.__dict__.copy()
        state.pop('_fd_engine', None)
        return state

    def forward(self, x):
        """CPU tensors (BASELINE config 1 plumbing) run on stock PyTorch, exactly like the reference (models.py:457-460).
        A CUDA tensor through the depthwise NNConv decoder ("MobileNet-NNConv5(dw)", reference README.md:37) takes the same
        fused sm_90a path as MobileNetSkipAdd, just without skips.  A CUDA fp16 / bf16 tensor through the dense decoder
        ("MobileNet-NNConv5", README.md:36) takes the engine too, with the decoder convs on conv_tc_kernel.  The DeConv and
        UpConv decoders route the same way as the dense NNConv decoder.

        An fp32 CUDA tensor through a dense decoder follows ``torch.get_float32_matmul_precision()``.  Under ``'high'`` or
        ``'medium'`` it takes the engine, whose decoder convs run as split TF32 on the tensor cores (three TF32 products
        per term, each within 3*2^-22 of the exact product), which keeps the result within the fp32 bound of 1e-3.  Under
        the default ``'highest'`` it stays on stock PyTorch.  The rule is the fp32 accuracy contract, not speed: stock
        PyTorch runs these convs under cuDNN's default TF32 conv precision, about 1e-2 away on the NNConv5 golden, and
        split TF32 is within the bound; a user who asks for ``'high'`` gets the faster, still fp32-accurate path.

        ``in_channels`` from 1 to 7 (depth only: 1, RGB-D: 4) routes the same way when ``x`` has that many channels; the
        engine's stem reads them all.  8 or more channels, or an input whose channel count differs from the stem's, stays
        on stock PyTorch (which raises for the latter)."""
        c_in = self.mobilenet[0][0].weight.shape[1]
        fused_ok = (x.is_cuda and not self.training and x.dim() == 4 and x.shape[1] == c_in and 1 <= c_in <= 7 and
                    x.shape[2] % 32 == 0 and x.shape[3] % 32 == 0)     # what the fused plan covers; anything else: stock PyTorch
        if fused_ok:
            from fastdepth_b200 import plan as _plan
            split_tf32 = torch.get_float32_matmul_precision() != 'highest'
            if _plan.supports(self) and not (x.dtype == torch.float32 and _plan.dense_decoder(self) and not split_tf32):
                engine = self.__dict__.get('_fd_engine')
                if engine is None:
                    from fastdepth_b200.engine import SkipAddEngine
                    engine = SkipAddEngine(self)
                    self.__dict__['_fd_engine'] = engine
                return engine(x)
        return self.decoder(self.mobilenet(x))


# --------------------------------------------------------------------------------------
# the hot path
# --------------------------------------------------------------------------------------
class MobileNetSkipAdd(nn.Module):
    """MobileNet encoder -> NNConv5(depthwise) decoder with additive skips.

    Drop-in for reference models.py:654-732.  ``widths`` (optional, an extension) is a
    pair ``(encoder_out[14], decoder_out[5])`` for NetAdapt-pruned variants; the
    released pruned checkpoint is a whole-module pickle (reference main.py:49-57) and
    simply carries its own Conv/BN shapes, which the plan builder reads.
    """

    def __init__(self, output_size, pretrained=True, widths=None):
        super().__init__()
        self.output_size = output_size
        enc_w, dec_w = (None, None) if widths is None else widths
        backbone = imagenet.mobilenet.MobileNet(widths=enc_w)
        if pretrained:
            _load_imagenet_encoder(backbone)
        else:
            backbone.apply(weights_init)
        for i in range(14):
            setattr(self, 'conv%d' % i, backbone.model[i])

        c = backbone.model[13][3].out_channels
        dec_w = tuple(dec_w) if dec_w is not None else tuple(c >> (j + 1) for j in range(5))
        kernel_size = 5
        for j, c_out in enumerate(dec_w):
            setattr(self, 'decode_conv%d' % (j + 1),
                    nn.Sequential(depthwise(c, kernel_size), pointwise(c, c_out)))
            c = c_out
        self.decode_conv6 = pointwise(c, 1)
        # The reference calls weights_init on the Sequential containers (models.py:699-704),
        # which matches none of its isinstance arms: decoder keeps PyTorch's default init.
        for j in range(1, 7):
            weights_init(getattr(self, 'decode_conv%d' % j))

    # the engine holds device pointers; never pickle / deepcopy it with the module
    def __getstate__(self):
        state = self.__dict__.copy()
        state.pop('_fd_engine', None)
        return state

    def forward(self, x):
        """One C-ABI call (``fd_forward``) on the caller's current CUDA stream.

        x: [N,3,H,W] CUDA tensor, fp32/fp16/bf16 (must match the module's parameter dtype),
        any strides; H, W multiples of 32.  In fp32 the pointwise convs follow ``torch.get_float32_matmul_precision()``:
        'highest' (the default) keeps them on fp32 SIMT kernels, 'high' / 'medium' runs them as split TF32 (three TF32
        products per term) on the tensor cores.  Returns a fresh contiguous [N,1,H,W] tensor of
        the same dtype/device (reference models.py:706-732 contract)."""
        engine = self.__dict__.get('_fd_engine')
        if engine is None:
            from fastdepth_b200.engine import SkipAddEngine
            engine = SkipAddEngine(self)
            self.__dict__['_fd_engine'] = engine
        return engine(x)


class MobileNetSkipConcat(MobileNetSkipAdd):
    """MobileNet encoder -> NNConv5(depthwise) decoder with CONCATENATED skips.

    Drop-in for reference models.py:734-814: same children (``conv0..conv13``, ``decode_conv1..6``) and ``state_dict``
    schema; decoder blocks 3, 4, 5 take ``cat(upsampled, skip)`` (512, 256, 128 input channels, reference l.769-777,
    806-811).  The forward is the same single C-ABI call; ``fastdepth_b200.plan`` marks the three skips as
    ``skip_mode = 1`` and the kernels write both halves of every concatenation into channel slices of one buffer."""

    def __init__(self, output_size, pretrained=True):
        super().__init__(output_size, pretrained)
        kernel_size = 5
        # (in, out) of decode_conv1..5 with the concatenated skips of conv5 (256), conv3 (128), conv1 (64)
        for j, (c_in, c_out) in enumerate(((1024, 512), (512, 256), (512, 128), (256, 64), (128, 32)), start=1):
            setattr(self, 'decode_conv%d' % j, nn.Sequential(depthwise(c_in, kernel_size), pointwise(c_in, c_out)))
        self.decode_conv6 = pointwise(32, 1)
