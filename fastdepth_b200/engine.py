"""Forward dispatch of ``models.MobileNetSkipAdd`` onto the C-ABI (one ``fd_forward`` per call).

Replaces the Python layer loop of reference models.py:706-732 and every PyTorch operator it
launches (SURVEY.md section 2b).  The engine is created lazily on the first forward so that
modules restored by ``torch.load`` without ``__init__`` (reference main.py:49-57) work.

fp32 inputs follow PyTorch's fp32 matmul precision: under ``torch.set_float32_matmul_precision('high')`` or ``'medium'``
the pointwise convs (1x1 convs are matmuls) and the convs of the dense decoders (NNConv5 / NNConv3, DeConv<k>, UpConv:
implicit GEMMs) run as split TF32 on the tensor cores (plan option ``tf32x3``, within 3*2^-22 of each exact product);
under the default ``'highest'`` they stay on the fp32 SIMT kernels.  An explicit ``set_option('tf32x3', v)`` wins over the
precision setting.  ``models.MobileNet`` hands an fp32 input with a dense decoder to the engine only under ``'high'`` or
``'medium'``: split TF32 stays within the fp32 bound of 1e-3 where cuDNN's plain TF32 convs do not.

One plan per (device, dtype) is live at a time.  A request [n,c_in,h,w] (c_in the stem's input channels, 1..7) whose pixels n*h*w fit the plan's capacity (the
n*h*w it was built for) runs on it, whatever its batch size and resolution (the C-ABI builds the steps for that shape once,
over the plan's buffers and weights; ``fd_forward_shape``).  A larger request replaces it with a plan built for the
request's own shape, whose capacity covers everything the old one served.  So an evaluation with a short last batch, or a
serving loop that sees many batch sizes and resolutions (224x224 and 480x640, say), holds one set of activation buffers
and packed weights instead of one per shape.
"""
import torch

from . import plan as _plan

_SUPPORTED = (torch.float32, torch.float16, torch.bfloat16)


class SkipAddEngine:
    def __init__(self, module):
        self.module = module
        self.plans = {}          # (device index, dtype) -> Plan (built for the largest n*h*w seen since the last refresh)
        self.signature = None
        self.options = {}

    # -- weight freshness ----------------------------------------------------------------------
    def _weights_signature(self):
        """Per-call freshness check over EVERY parameter and buffer of the module: storage pointer, dtype and the
        autograd version counter (bumped by every in-place write through the tensor itself: ``load_state_dict``,
        ``p.copy_`` / ``p.mul_`` under ``no_grad``, optimizer steps).  ~250 tensors, a few tens of microseconds; catches
        .cuda()/.half()/.to() too.  Writes that bypass the counter (``p.data.mul_()``, a raw pointer handed to another
        library) still need an explicit ``refresh()``."""
        sig = []
        for t in self.module.parameters():
            sig.append((t.data_ptr(), t.dtype, t._version))
        for t in self.module.buffers():
            sig.append((t.data_ptr(), t.dtype, t._version))
        return tuple(sig)

    def refresh(self):
        """Drop packed weights (call after editing parameters in place)."""
        for p in self.plans.values():
            p.close()
        self.plans.clear()
        self.signature = None

    def set_option(self, name, value):
        """Forwarded to ``fd_plan_set_option`` on every current and future plan."""
        prev = self.options.get(name)
        self.options[name] = int(value)
        try:
            for p in self.plans.values():
                p.set_option(name, value)
        except Exception:
            if prev is None:
                self.options.pop(name, None)
            else:
                self.options[name] = prev
            raise

    # -- forward ---------------------------------------------------------------------------------
    def plan_for(self, x, exact=False):
        """The plan that runs ``x``: the live plan of its (device, dtype) if the pixels of ``x`` (n*h*w) fit its capacity
        (``exact``: its own (n, h, w) equals that of ``x``, as the host pipeline needs), else a new plan built for the shape
        of ``x`` that replaces it."""
        m = self.module
        if m.training:
            raise RuntimeError("fastdepth_b200 is inference-only: call model.eval() first "
                               "(BatchNorm is folded from running statistics, reference main.py:65)")
        if not x.is_cuda:
            raise RuntimeError("fastdepth_b200: the accelerated forward needs a CUDA tensor; "
                               "there is no CPU fallback (use models.MobileNet for CPU plumbing)")
        stem_w = _plan._blocks_of(m)[0][0][0].weight
        if x.dim() != 4:
            raise RuntimeError("expected input [N,%d,H,W], got %s" % (stem_w.shape[1], tuple(x.shape)))
        if x.shape[1] != stem_w.shape[1]:
            raise RuntimeError("Given groups=1, weight of size %s, expected input%s to have %d channels, but got %d channels "
                               "instead" % (list(stem_w.shape), list(x.shape), stem_w.shape[1], x.shape[1]))
        wdtype = stem_w.dtype
        if x.dtype != wdtype:
            raise RuntimeError("Input type (%s) and weight type (%s) should be the same" % (x.dtype, wdtype))
        if x.dtype not in _SUPPORTED:
            raise RuntimeError("unsupported dtype %s" % x.dtype)
        n, _, h, w = x.shape
        if h % 32 or w % 32:
            raise RuntimeError("The size of tensor a must match the size of tensor b: H and W must be multiples "
                               "of 32 for the skip connections to line up, got %dx%d" % (h, w))
        sig = self._weights_signature()
        if sig != self.signature:
            self.refresh()
            self.signature = sig
        key = (x.device.index, x.dtype)
        p = self.plans.get(key)
        if p is not None and (n * h * w > p.n * p.h * p.w or (exact and (n, h, w) != (p.n, p.h, p.w))):
            del self.plans[key]       # freed with its last reference (a pending host-pipeline ticket holds one)
            p = None
        if p is None:
            p = _plan.Plan.from_module(m, n, h, w, x.dtype, x.device.index)
            try:
                for k, v in self.options.items():
                    p.set_option(k, v)
            except Exception:
                p.close()                      # an option stored before any plan existed turned out to be invalid
                raise
            self.plans[key] = p
        if x.dtype == torch.float32 and 'tf32x3' not in self.options:
            want = int(torch.get_float32_matmul_precision() != 'highest')
            if p.get_option('tf32x3') != want:
                p.set_option('tf32x3', want)       # the steps are rebuilt on the next forward
        return p

    def __call__(self, x):
        p = self.plan_for(x)
        xc = x if x.is_contiguous() else x.contiguous()
        y = torch.empty((x.shape[0], 1, x.shape[2], x.shape[3]), dtype=x.dtype, device=x.device)
        p.forward(xc, y, torch.cuda.current_stream(x.device).cuda_stream)
        return y


class ForwardLanes:
    """Throughput front end: ``lanes`` independent copies of the forward plan -- each with its own activation buffers, its own
    CUDA stream and its own C-ABI host pipeline (``fd_pipeline_submit`` / ``fd_pipeline_wait``) -- that take batches round-robin.

    One forward is a chain of 18 kernels, most of them persistent with one 227 KB CTA per SM, so at every kernel boundary the SMs that finish early
    idle until the next kernel has filled its pipeline.  A second and third batch in flight
    on other streams fill those gaps with their own kernels.
    The module's own ``forward`` keeps strict single-stream semantics (and the lowest latency); this class is for serving loops that
    have several batches to run and only care when each one is done.  (Programmatic dependent launch stays off on the lanes: its
    early-launched dependents hold SMs that another lane's kernel could use.)
    """

    def __init__(self, module, lanes=3, options=None):
        if lanes < 1:
            raise ValueError("lanes must be >= 1")
        self.engines = [SkipAddEngine(module) for _ in range(lanes)]
        opts = dict(options or {})
        if lanes > 1:
            opts.setdefault('pdl', 0)
        for e in self.engines:
            for k, v in opts.items():
                e.set_option(k, v)
        self.streams = {}            # device index -> [torch.cuda.Stream] * lanes
        self.next = 0

    def __len__(self):
        return len(self.engines)

    def streams_for(self, device):
        """The lanes' CUDA streams on ``device`` (created on first use)."""
        return self._streams(device)

    def _streams(self, device):
        s = self.streams.get(device.index)
        if s is None:
            s = [torch.cuda.Stream(device=device) for _ in self.engines]
            self.streams[device.index] = s
        return s

    def plans_for(self, x):
        return [e.plan_for(x) for e in self.engines]

    def forward(self, x, y=None):
        """Enqueue one forward of ``x`` ([N,3,H,W], CUDA, contiguous) on the next lane; returns ``(y, done)`` where ``done`` is a CUDA
        event recorded after the forward on the lane's stream.  ``x`` must be ready on the caller's current stream (the lane waits for
        it); consume ``y`` after ``done.synchronize()`` or ``torch.cuda.current_stream().wait_event(done)``."""
        lane = self.next
        self.next = (self.next + 1) % len(self.engines)
        p = self.engines[lane].plan_for(x)
        st = self._streams(x.device)[lane]
        if y is None:
            y = torch.empty((x.shape[0], 1, x.shape[2], x.shape[3]), dtype=x.dtype, device=x.device)
        st.wait_stream(torch.cuda.current_stream(x.device))
        x.record_stream(st); y.record_stream(st)
        p.forward(x if x.is_contiguous() else x.contiguous(), y, st.cuda_stream)
        done = torch.cuda.Event()
        done.record(st)
        return y, done

    def submit(self, x_host, y_host, like):
        """Host pipeline: H2D of the pinned batch, forward, D2H of the depth maps, all asynchronous, on the next lane.  ``like`` is any
        CUDA tensor of the batch's shape/dtype (selects the plan).  Returns a handle for ``wait``."""
        lane = self.next
        self.next = (self.next + 1) % len(self.engines)
        p = self.engines[lane].plan_for(like, exact=True)      # the host pipeline moves the plan's full batch
        return lane, p, p.pipeline_submit(x_host, y_host)

    @staticmethod
    def wait(handle):
        _, p, ticket = handle
        p.pipeline_wait(ticket)

    def synchronize(self):
        for ss in self.streams.values():
            for s in ss:
                s.synchronize()
