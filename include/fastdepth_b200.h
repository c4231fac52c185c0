/*
 * fastdepth_b200 -- C-ABI of the H100-native FastDepth forward path.
 *
 * This is the drop-in boundary for ONE hot path of dwofk/fast-depth:
 *     MobileNetSkipAdd.forward            (reference models.py:706-732)
 * i.e. the MobileNet encoder (reference imagenet/mobilenet.py:22-54), the NNConv5
 * depthwise-separable decoder with 2x nearest upsampling and additive skips
 * (reference models.py:61-75, 683-698, 720-731), plus the per-image depth metrics the
 * only caller computes on the result (reference metrics.py:31-55 via main.py:80-82).
 *
 * The reference has no FFI of its own (it is pure Python on PyTorch); the entry points
 * below are what a binding for this path binds.  The repo's own binding is
 * fastdepth_b200/_lib.py (ctypes); INTEGRATION.md shows the reference-side stub.
 *
 * Conventions
 *   - plain C: opaque handle, ints, raw pointers; no C++/torch types cross the boundary.
 *   - every function returns 0 on success, a negative fd_status otherwise; the message is
 *     retrievable (thread-local) with fd_last_error().  No C++ exception crosses the ABI.
 *   - "dev" pointers are CUDA device pointers on the plan's device, "host" pointers are
 *     ordinary (ideally pinned) host memory.  `stream` is a cudaStream_t passed as void*.
 *   - all work is stream-ordered and asynchronous unless stated otherwise.
 *   - a plan is not thread-safe; use one plan per (device, N, H, W, dtype) per thread.
 *   - there is NO CPU fallback: without a CUDA device every call fails with FD_ERR_CUDA.
 */
#ifndef FASTDEPTH_B200_H
#define FASTDEPTH_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FD_ABI_VERSION 2

typedef struct fd_plan fd_plan;

typedef enum {
    FD_OK = 0,
    FD_ERR_INVALID = -1,      /* bad argument / unsupported shape (H or W % 32, C % 8 ...)   */
    FD_ERR_CUDA = -2,         /* CUDA runtime / driver error, or no device                   */
    FD_ERR_STATE = -3,        /* call order violated (weights missing, plan destroyed ...)   */
    FD_ERR_UNSUPPORTED = -4   /* valid request this build has no kernel for                  */
} fd_status;

/* storage + arithmetic type of activations and of the pointwise contraction inputs;
 * accumulation, BN scale/bias and activations are always computed in fp32.
 * (reference: dtype of the tensor handed to model(input), main.py:68,74-75) */
typedef enum { FD_F32 = 0, FD_F16 = 1, FD_BF16 = 2 } fd_dtype;

typedef enum {
    FD_STAGE_STEM = 0,   /* dense 3x3 stride-s conv + BN + act, NCHW in -> NHWC out
                            (conv_bn, reference imagenet/mobilenet.py:22-27)                 */
    FD_STAGE_DWPW = 1,   /* depthwise kxk(stride) + BN + act -> pointwise 1x1 + BN + act
                            (conv_dw, reference imagenet/mobilenet.py:29-38;
                             depthwise+pointwise, reference models.py:61-75, 683-697)        */
    FD_STAGE_HEAD = 2,   /* pointwise C->1 + BN + act, NHWC in -> [N,1,H,W] out
                            (decode_conv6, reference models.py:698, 731)                     */
    FD_STAGE_CONV = 3,   /* dense kxk (k in {3,5}) stride-1 conv, padding (k-1)/2, + BN + act, then the
                            optional nearest x2 upsample; NHWC in -> NHWC out.  No skip, no stride 2
                            (conv() blocks of the dense NNConv decoder, reference models.py:52-59, 245-270) */
    FD_STAGE_DECONV = 4, /* ConvTranspose2d(c_in, c_out, k, stride 2, padding (k-1)/2, output_padding 1), k in
                            {3,5,7,9}, + BN + act; NHWC [N,h,w,c_in] in -> NHWC [N,2h,2w,c_out] out.  stride must
                            be 2, upsample 0, skip_src -1 (convt() blocks of the DeConv decoder, reference
                            models.py:77-87, 145-180) */
    FD_STAGE_UPCONV = 5  /* 2x2 zero-insertion unpool, then a 5x5 stride-1 conv with padding 2, + BN + act;
                            NHWC [N,h,w,c_in] in -> NHWC [N,2h,2w,c_out] out.  ksize 5, stride 2, upsample 0,
                            skip_src -1 (upconv() blocks of the UpConv decoder, reference models.py:18-34,
                            101-107, 183-201) */
} fd_stage_kind;

typedef enum { FD_ACT_RELU = 0, FD_ACT_RELU6 = 1 } fd_act;

typedef struct {
    int32_t kind;        /* fd_stage_kind                                                    */
    int32_t c_in;        /* input channels; the stem's is x's: 1..7 (3 RGB, 1 depth, 4 RGB-D) */
    int32_t c_out;       /* output channels (1 for the head)                                 */
    int32_t ksize;       /* spatial kernel: 3 (stem, encoder dw), 5 (decoder dw), 1 (head)   */
    int32_t stride;      /* stride of the spatial conv (1 or 2)                              */
    int32_t act;         /* fd_act applied after BOTH halves (encoder ReLU6, decoder ReLU)   */
    int32_t upsample;    /* 1: output is 2x nearest-upsampled (F.interpolate, models.py:723) */
    int32_t skip_src;    /* stage index whose output is combined with this stage's upsampled
                            output (models.py:724-729 / 806-811), or -1                      */
    int32_t skip_mode;   /* 0: ADD (MobileNetSkipAdd, models.py:724-729); 1: CONCATENATE along
                            channels, upsampled output first (MobileNetSkipConcat,
                            models.py:806-811) -- the next stage then has c_in = c_out + c_skip  */
} fd_stage_desc;

/* Build a plan for a stage list (always: 1 STEM, k stages each DWPW, CONV, DECONV or UPCONV, 1 HEAD) at a fixed problem size.
 * Allocates NHWC activation buffers and packed-weight storage on `device`.
 * H and W must be multiples of 32 (reference forward's skip shapes only line up then),
 * every c_in/c_out except the stem's c_in and the head's c_out a multiple of 8.  The stem's c_in is the channel count of x:
 * 1..7 (x is [N,c_in,H,W]; K = 9 c_in fits one 64-element K row of the tensor-core stem).  c_in <= 0 fails with
 * FD_ERR_INVALID, c_in >= 8 with FD_ERR_UNSUPPORTED. */
int fd_plan_create(const fd_stage_desc* stages, int n_stages,
                   int n, int h, int w, int dtype /* fd_dtype */, int device, fd_plan** out);

/* Upload one stage's parameters (HOST pointers, fp32, BatchNorm already folded to a
 * per-channel affine y = conv * scale + bias by the caller; folding is exact in fp32,
 * reference BN eval formula, eps 1e-5).  Synchronous.  May be called again after a
 * parameter update.
 *   STEM : dw_* = NULL ; pw_w = [c_out][c_in][k][k]  ; pw_scale/pw_bias = [c_out]
 *   DWPW : dw_w = [c_in][k][k], dw_scale/dw_bias = [c_in] ; pw_w = [c_out][c_in], pw_scale/pw_bias = [c_out]
 *   CONV : dw_* = NULL ; pw_w = [c_out][c_in][k][k]  ; pw_scale/pw_bias = [c_out]  (PyTorch's layout; the
 *          plan keeps it as [c_out][k*k][c_in] in the plan dtype, the K-major operand both conv kernels read)
 *   DECONV: dw_* = NULL ; pw_w = [c_in][c_out][k][k] (PyTorch's ConvTranspose2d layout) ; pw_scale/pw_bias = [c_out]
 *   UPCONV: dw_* = NULL ; pw_w = [c_out][c_in][5][5] ; pw_scale/pw_bias = [c_out]
 *          (both are kept as [c_out][k*k][c_in], the taps grouped by output phase, i.e. by the parity of the output pixel)
 *   HEAD : dw_* = NULL ; pw_w = [1][c_in]            ; pw_scale/pw_bias = [1]              */
int fd_plan_set_stage_weights(fd_plan* plan, int stage,
                              const float* dw_w, const float* dw_scale, const float* dw_bias,
                              const float* pw_w, const float* pw_scale, const float* pw_bias);

/* Tunables, by name.  Unknown names fail with FD_ERR_INVALID.
 *   "path"       0 = SIMT reference-quality kernels (all dtypes), 1 = fused wgmma block
 *                kernels where available (16-bit dtypes)            [default 1]
 *   "fold_head"  1 = apply decode_conv6 below the last upsample (exact: 1x1 conv/BN/ReLU
 *                commute with nearest upsampling, SURVEY.md section 2b row 8) [default 1]
 *   "graph"      1 = replay fd_forward from a captured CUDA graph   [default 1]
 *   "tma_epilogue" 1 = fused blocks write their output tiles with TMA tensor stores  [default 1]
 *   "inplace_skip" 1 = decoder blocks ADD their upsampled output into the skip tensor in place
 *                (TMA reduce-add); the skip source's stage buffer then holds the decoder output
 *                after fd_forward (set 0 for stage-by-stage inspection)  [default 1]
 *   "pdl"        1 = tensor-core kernels are launched with programmatic dependent launch so that each
 *                kernel's prologue overlaps the previous kernel's tail.  With one 227 KB CTA per SM the early-launched
 *                dependents mostly hold SMs idle while they wait for the previous grid  [default 0]
 *   "chain"      1 = a run of consecutive 3x3 stride-1 blocks on a small feature map (conv7..conv11 at 14x14) executes as ONE
 *                kernel on 2-CTA clusters with every intermediate activation resident in shared memory; the intermediate
 *                stages' buffers are then not written (set 0 for stage-by-stage inspection)  [default 1]
 *   "cluster"    1 = the block planner may run a block on thread-block clusters of 2 or 4 CTAs that share one 128-pixel tile:
 *                each CTA computes the depthwise half of a quarter (half) of the K-blocks, broadcasts its operand tiles to
 *                the others through distributed shared memory and runs the MMAs of one output-channel split (chosen by
 *                the planner's cost model for the small-map, many-channel blocks)  [default 1]
 *   "tf32x3"     1 = in an fp32 plan on path 1, the pointwise half of every DWPW stage runs on the tensor cores as split
 *                TF32: each operand is split into a TF32 high part and a TF32 low part (round to nearest), and each
 *                product is a_lo*b_hi + a_hi*b_lo + a_hi*b_hi in an fp32 accumulator, within 3*2^-22 of the exact
 *                product (plain TF32: about 2^-11).  The depthwise half, stem and head keep their fp32 SIMT kernels;
 *                "chain" and "cluster" do not apply.  16-bit plans and path 0 ignore it.  fd_stage_buffer(which = 1)
 *                still returns the depthwise intermediate.  (fastdepth_b200.engine sets it from
 *                torch.get_float32_matmul_precision())  [default 0]
 *   "unfuse"     a 16-bit DWPW stage on path 1 may run as two steps instead of the fused block kernel: dw_mid_kernel writes the
 *                depthwise half once to the stage's intermediate, and conv_tc_kernel runs the pointwise half over it as a
 *                1x1 conv (a skip is reduce-added in place).  The result is the fused kernel's, bit for bit.
 *                0 = never; 1 = the stages the block planner would split 8 ways or more over the output channels, or run
 *                on a tile-sharing cluster, and whose intermediate is at most 16 MB (stock b64 224x224: conv12, conv13,
 *                decode_conv1); 2 = every DWPW stage the 1x1 step supports (not the block with the folded head, not a
 *                stage inside a chain, a skip only with "tma_epilogue" and "inplace_skip").  A stage whose block-kernel
 *                plan is pinned by FD_TC_MAX_NCTA, FD_TC_CLUSTER >= 2, FD_TC_WMC or FD_TC_DW_TEAMS stays fused.
 *                fd_stage_buffer(which = 1) returns the intermediate of a two-step stage.  [default 1]
 *   "front"      1 = in a 16-bit plan on path 1 the stem and the two DWPW stages after it run as ONE kernel
 *                (front_tc_kernel) when they have the stock MobileNet shapes: stem 3 -> 32 stride 2 with ReLU6, 3x3
 *                blocks 32 -> 64 stride 1 and 64 -> 128 stride 2 with one act, no skip, no concatenation onto their
 *                outputs.  An item is an 8x8 tile of conv2's output; the conv0 and conv1 pixels it needs are computed in
 *                shared memory and each stage's own part is written to its buffer, so conv0 and conv1 are never read back.
 *                The result is the three kernels', bit for bit.  0 = three steps.  [default 1]
 *   "wait_sleep_ns" > 0: latency-tolerant roles of the fused block kernel (the TMA producer waiting for a
 *                free stage) sleep this many ns between barrier
 *                probes instead of spinning (the spinning waiters do not
 *                take issue slots the depthwise warps could use)  [default 0]   */
int fd_plan_set_option(fd_plan* plan, const char* name, int value);
int fd_plan_get_option(fd_plan* plan, const char* name, int* value);

/* The hot path.  x_dev: [N,c_in,H,W] contiguous, plan dtype, c_in the stem's.  y_dev: [N,1,H,W] contiguous,
 * plan dtype.  Enqueues on `stream`; returns without synchronising.  A plan owns one set of activation
 * buffers: calls on different streams are ordered after each other by an event (never corrupted, never
 * overlapped); to keep several forwards in flight use several plans (one per stream).
 * Replaces: pred = model(input)  (reference main.py:74-75 -> models.py:706-732). */
int fd_forward(fd_plan* plan, const void* x_dev, void* y_dev, void* stream);

/* The same forward over the first n images, 1 <= n <= the plan's N, at the plan's own H x W: fd_forward_shape(plan, n, H,
 * W, ...).  x_dev is [n,c_in,H,W] and y_dev [n,1,H,W]. */
int fd_forward_batch(fd_plan* plan, int n, const void* x_dev, void* y_dev, void* stream);

/* The forward of n images at any resolution h x w that fits the plan's pixel capacity: x_dev is [n,c_in,h,w] (c_in the stem's) and y_dev
 * [n,1,h,w], contiguous, plan dtype.  Accepted: n >= 1, h and w positive multiples of 32, n*h*w <= N*H*W (every stage
 * buffer of the plan is dense NHWC of N*(H/s)*(W/s)*C elements, so the request fits in its front).  Anything else fails
 * with FD_ERR_INVALID; for a request that does not fit, the message names the capacity in pixels and the plan's (N, H, W).
 * Nothing is read or written past n*h*w elements of x_dev (times c_in) or y_dev.  The result equals that of a plan built for
 * (n, h, w), bit for bit.  The plan builds the steps for (n, h, w) on first use (every stage's geometry, planner choices,
 * grids, tensor maps, whether a run of blocks takes the chain kernel) over its own activation buffers, packed weights and
 * split weights; it keeps up to 8 such step sets, least recently used first out (the set of its own (N, H, W) is always
 * kept), and captures graphs per (x_dev, y_dev, n, h, w).  fd_forward(plan, ...) is fd_forward_shape(plan, N, H, W, ...).
 * fd_forward_host and fd_pipeline_* always run N images at H x W, and copy N*c_in*H*W elements of x. */
int fd_forward_shape(fd_plan* plan, int n, int h, int w, const void* x_dev, void* y_dev, void* stream);

/* Same, end to end from HOST buffers: H2D copy of x, forward, D2H copy of y, then waits for
 * the stream.  (reference main.py:68 input.cuda() ... main.py:85-98 pred.cpu()) */
int fd_forward_host(fd_plan* plan, const void* x_host, void* y_host, void* stream);

/* Pipelined end-to-end evaluation from HOST buffers (what the reference's DataLoader(pin_memory) + input.cuda()
 * + pred.cpu() loop does, main.py:40-41, 68, 85-98, with the copies overlapped): submit() enqueues the upload of
 * x_host (pinned), the forward and the download into y_host (pinned) on the plan's own three streams and returns
 * a ticket at once; up to 3 batches are in flight (submit blocks on the oldest when all slots are busy).
 * wait(ticket) returns when y_host holds that batch's depth maps.  Tickets complete in order. */
int fd_pipeline_submit(fd_plan* plan, const void* x_host, void* y_host, unsigned long long* ticket);
int fd_pipeline_wait(fd_plan* plan, unsigned long long ticket);

/* Introspection for stage-parity tests: the NHWC buffer stage `stage` wrote in the last
 * fd_forward (valid until the next one).  c_stride = elements between pixels.
 * which = 0: the stage output (after upsample/skip-add); 1: the depthwise intermediate
 * (only materialised on path 0 and by the two-step stages of "unfuse"; a CONV, DECONV or UPCONV stage has none and fails with FD_ERR_INVALID). */
int fd_stage_buffer(fd_plan* plan, int stage, int which, void** dev_ptr,
                    int* n, int* h, int* w, int* c, int* c_stride);

/* Bookkeeping used by bench.py.  A "step" is one kernel launch of fd_forward under the current
 * options (a DWPW stage is one fused step on path 1, or two under "unfuse"; a dw + a pw step on path 0); the step functions, fd_plan_time_steps,
 * fd_plan_trace_stage and fd_stage_buffer describe the steps of the plan's own (N, H, W).  The workspace bytes include, once
 * the steps are built, the device memory they hold: with "tf32x3", the split weights [2][c_out][k*k][c_in] fp32 of every
 * split-TF32 step (once, shared by every shape), and the packed parameter copies of every step set fd_forward_shape
 * built for a shape other than (N, H, W). */
int fd_plan_launches_per_forward(fd_plan* plan, int* n_launches);
int fd_plan_workspace_bytes(fd_plan* plan, size_t* bytes);
int fd_plan_step_count(fd_plan* plan, int* n_steps);
/* Stage index, ALGORITHMIC bytes (external inputs once + outputs once + weights once; SURVEY.md
 * section 8d) and MACs of step `step`, plus its kernel name. */
int fd_plan_step_info(fd_plan* plan, int step, int* stage, double* alg_bytes, double* macs,
                      char* kernel_name, int name_cap);
/* The same step's MACs split by the pipe that executes them: depthwise taps (channel-wise, SIMT FMA pipe; north_star keeps
 * them off the tensor cores) and the dense contractions (stem im2col, pointwise 1x1, head; tensor pipe on path 1).  bench.py
 * turns them into the per-stage FMA-pipe and tensor-pipe floors it prints next to the HBM floor. */
int fd_plan_step_macs(fd_plan* plan, int step, double* dw_macs, double* dense_macs);
/* Time every step's kernel alone with CUDA events on `stream` (`warmup` + `iters` launches each;
 * a 256 MB buffer is written between launches when flush_l2 != 0 so inputs come from HBM).
 * ms_out[n_steps] = mean launch duration.  Synchronous. */
int fd_plan_time_steps(fd_plan* plan, const void* x_dev, void* y_dev, void* stream,
                       int warmup, int iters, int flush_l2, float* ms_out);

/* Debug: run stage `stage`'s fused block kernel once with its in-kernel timeline enabled and return
 * the SM-clock stamps of CTA 0: rows = {TMA issue, dw start, dw math done, A tile published, MMA
 * operands ready, MMA issued, epilogue start, epilogue done}, one column per K-block / item.
 * The previous fd_forward's activations are reused as inputs. Synchronous. */
int fd_plan_trace_stage(fd_plan* plan, int stage, void* y_dev, void* stream,
                        unsigned long long* out_host, int cap, int* rows, int* cols);

/* Debug (host only, needs no GPU): the shared-memory / pipeline plan the fused block kernel would use for one
 * block.  out[0..15] = {ok, splits, n_cta, items, kblocks, s_in, s_a, s_b, bn, nb, b_resident, n_stg, smem_bytes,
 * in_stage_stride, cs (cluster size: CTAs sharing one tile's depthwise half), dw_teams}.  cap must be at least 16. */
int fd_debug_block_plan(int ksize, int stride, int h_out, int w_out, int n, int c_in, int c_out, int head,
                        int* out, int cap);

/* Debug (host only, needs no GPU): the tile plan of the dense conv kernel (conv_tc_kernel) for one CONV stage on
 * `n_sms` SMs.  out[0..15] = {ok, ni, th, tw (tile = ni images x th rows x tw columns = 128 output pixels), bn (output
 * channels per item), stages (operand ring depth), m_tiles, n_splits, items, waves, kblocks (64-channel blocks per
 * tap), smem_bytes, useful_rows_permille, cost (modelled time, arbitrary units), 0, 0}.  cap must be at least 16. */
int fd_debug_conv_plan(int ksize, int h_out, int w_out, int n, int c_in, int c_out, int n_sms, int* out, int cap);

/* Debug (host only, needs no GPU): the same plan for a DECONV or UPCONV stage (`kind`) on an h_in x w_in input map: four
 * stride-1 phase convs at the input resolution, items = m_tiles * n_splits * phase groups.  out[0..15] as in
 * fd_debug_conv_plan except out[14] = the number of phase groups (4: one phase per item, 2: the diagonal pairs {00, 11} and
 * {01, 10}); out[16 + 5 q .. 20 + 5 q] = {tap0, ny, nx, dy0, dx0} of phase q = 2 ry + rx (its taps tap0 .. tap0 + ny nx - 1
 * of the repacked weights, input offsets dy0 .. dy0 + ny - 1 by dx0 .. dx0 + nx - 1); out[36 + 2 g .. 37 + 2 g] = the phases
 * of group g (-1 = none), in execution order.  cap must be at least 44. */
/* Debug (host only, needs no GPU): the tile plan of the split-TF32 pointwise step ("tf32x3") of one fp32 DWPW stage on an
 * h_out x w_out map (upsample: its output is stored through the four views of the 2x map).  out[0..13] as in
 * fd_debug_conv_plan, with kblocks counting 32-channel blocks (one 128-byte row of fp32); out[14] = bytes of one operand
 * stage (16 KB of A + 2 x bn x 128 B of B, the weights' high and low parts), out[15] = 0.  cap must be at least 16. */
int fd_debug_pw_tf32x3_plan(int h_out, int w_out, int n, int c_in, int c_out, int upsample, int n_sms, int* out, int cap);

/* Debug (host only, needs no GPU): the tile plan of the 16-bit pointwise step ("unfuse") of one DWPW stage on an h_out x w_out
 * map.  Without an upsample the n * h_out * w_out rows are planned as one image of rows / 16 x 16 pixels when 16 divides
 * them.  out[0..13] as in fd_debug_conv_plan (kblocks of 64 channels); out[14] = bytes of one operand stage (16 KB of A +
 * bn x 128 B of B), out[15] = 0.  cap must be at least 16. */
int fd_debug_pw_plan(int h_out, int w_out, int n, int c_in, int c_out, int upsample, int n_sms, int* out, int cap);

/* Debug (host only, needs no GPU): whether a 16-bit plan on path 1 of these stages at n x h x w runs its stem and the two
 * blocks after it as one front_tc_kernel step ("front"), and that kernel's budget.  out[0] = 1 when it does, out[1] = its
 * items (8x8 tiles of conv2's map, 0 when it does not), out[2] = dynamic shared memory per CTA in bytes, out[3] = CTAs per
 * SM, out[4] = threads per CTA, out[5..7] = bytes of its weight + parameter, A-operand and tile regions.  The budget is the
 * one for the stem's c_in: the x box holds c_in planes, c_in <= 3 fit inside the A region, c_in = 4 grows it by 2688 bytes
 * and c_in >= 5 would leave one CTA per SM, so the route is taken for c_in 1..4 only.  cap >= 8. */
int fd_debug_front_plan(const fd_stage_desc* stages, int n_stages, int dtype, int n, int h, int w, int* out, int cap);

int fd_debug_convt_plan(int kind, int ksize, int h_in, int w_in, int n, int c_in, int c_out, int n_sms, int* out, int cap);

/* Debug (host only, needs no GPU): the tile plan of the split-TF32 step ("tf32x3") of one dense fp32 stage: kind
 * FD_STAGE_CONV (ksize 1, 3 or 5; h x w = the conv resolution, upsample: the output goes through the four views of the 2x
 * map), FD_STAGE_DECONV (ksize 3, 5, 7 or 9) or FD_STAGE_UPCONV (ksize 5) on an h x w input map.  out[0..13] as in
 * fd_debug_conv_plan, with kblocks counting 32-channel blocks per tap; out[14] = bytes of one operand stage (16 KB of A +
 * 2 x bn x 128 B of B), out[15] = the number of phase groups (items = m_tiles * n_splits * groups); out[16..43] the phase
 * table and groups as in fd_debug_convt_plan (a CONV stage: phase 0 only).  cap must be at least 44. */
int fd_debug_conv_tf32x3_plan(int kind, int ksize, int h, int w, int n, int c_in, int c_out, int upsample, int n_sms,
                              int* out, int cap);

/* Per-image depth metrics on device (reference metrics.py:31-55 applied per image, as
 * main.py:40-41,80-82 does at batch size 1).  pred: [n, hw] of `dtype`; target: [n, hw] fp32.
 * Adds, for each image, its 10 metric values into sums_dev[0..9] (order: irmse, imae, mse,
 * rmse, mae, absrel, lg10, delta1, delta2, delta3) and 1.0 into sums_dev[10] (count), all
 * double (reference AverageMeter, metrics.py:71-95).  The cross-GPU reduction of that
 * 11-vector is the caller's single all-reduce (SURVEY.md section 8e). */
int fd_metrics_accumulate(const void* pred_dev, const float* target_dev, int dtype, int n, int hw,
                          double* sums_dev, int device, void* stream);

/* NYU-Depth-v2 validation pre-processing as ONE gather launch (reference dataloaders/nyu.py:48-59: Resize(250/480) ->
 * CenterCrop(228x304) -> Resize(out), all nearest-neighbour, rgb / 255; dataloaders/dataloader.py:90-111: HWC -> CHW).
 * rgb_dev: [n, h_in, w_in, 3] uint8; depth_dev: [n, h_in, w_in] float or NULL; rows_dev[out_h] / cols_dev[out_w]: the
 * composed source-index tables (fastdepth_b200/preprocess.py builds them from PIL's own nearest resize);
 * x_dev: [n, 3, out_h, out_w] of `dtype`; target_dev: [n, 1, out_h, out_w] float or NULL (with depth_dev). */
int fd_nyu_val_gather(const uint8_t* rgb_dev, const float* depth_dev, const int* rows_dev, const int* cols_dev,
                      int n, int h_in, int w_in, int out_h, int out_w, int dtype,
                      void* x_dev, float* target_dev, int device, void* stream);

void fd_plan_destroy(fd_plan* plan);

/* Thread-local message of the last failing call on this thread ("" if none). */
const char* fd_last_error(void);
int fd_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* FASTDEPTH_B200_H */
