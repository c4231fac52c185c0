// C-ABI of fastdepth_b200 (see include/fastdepth_b200.h): plan construction, weight packing,
// forward dispatch, stage timing.  Host-side C++; kernels live in the sibling .cu files.
#include <algorithm>
#include <cstring>
#include <functional>
#include <string>
#include <vector>

#include "fd_block_plan.h"
#include "fd_conv_plan.h"
#include "fd_common.cuh"

namespace fd {

BlockPlanOut block_tc_debug_plan(int ksize, int stride, int h_out, int w_out, int n, int c_in, int c_out, int head);
ConvPlanOut conv_tc_debug_plan(int kind, int ksize, int h_out, int w_out, int n, int c_in, int c_out, int n_sms);
ConvPlanOut pw_tf32x3_debug_plan(int h_out, int w_out, int n, int c_in, int c_out, int upsample, int n_sms);
ConvPlanOut pw_tc_debug_plan(int h_out, int w_out, int n, int c_in, int c_out, int upsample, int n_sms);
ConvPlanOut conv_tc_tf32x3_debug_plan(int kind, int ksize, int h_out, int w_out, int n, int c_in, int c_out, int upsample,
                                      int n_sms);

// ---- error state -----------------------------------------------------------------------
static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }
int fail(int code, const std::string& msg) {
    g_last_error = msg;
    return code;
}

// ---- kernels (fd_kernels_simt.cu, fd_block_tc.cu, fd_metrics.cu) -----------------------------
int launch_stem(int dtype, const void* x, void* out, const float* w, const float* scale, const float* bias,
                const StageGeom& g, cudaStream_t st);
int launch_dw(int dtype, const BlockArgs& a, cudaStream_t st);
int launch_pw(int dtype, const BlockArgs& a, cudaStream_t st);
int launch_conv(int dtype, const void* in, const void* w, void* out, const float* scale, const float* bias, const StageGeom& g,
                cudaStream_t st);
int launch_convt(int dtype, int kind, const void* in, const void* w, void* out, const float* scale, const float* bias,
                 const StageGeom& g, cudaStream_t st);
int launch_head(int dtype, const void* in, void* out, const float* w, float scale, float bias, long long m_total, int c,
                int in_pitch, int h, int wd, int up, int act, cudaStream_t st);
int launch_metrics(int dtype, const void* pred, const float* target, int n, int hw, double* sums, cudaStream_t st);
int launch_nyu_val_gather(int dtype, const uint8_t* rgb, const float* depth, const int* rows, const int* cols, int n, int h_in,
                          int w_in, int oh, int ow, void* x, float* t, cudaStream_t st);
// fused wgmma block kernel
struct BlockTcPlan;   // opaque per-stage state (tensor maps, tile config)
bool block_tc_supported(int dtype, const StageGeom& g, bool head_fused);
int block_tc_prepare(int dtype, const BlockArgs& a, const float* head_w, float head_scale, float head_bias, int head_act,
                     void* head_out, bool tma_epilogue, const TcLaunchOpts& opts, BlockTcPlan** out);
int block_tc_launch(BlockTcPlan* p, cudaStream_t st, void* head_out);
void block_tc_destroy(BlockTcPlan* p);
const char* block_tc_name(BlockTcPlan* p);
int block_tc_trace(BlockTcPlan* bp, cudaStream_t st, void* head_out, unsigned long long* out_host, int* rows, int* cols);
// fused multi-layer chain kernel (fd_chain_tc.cu): a run of 3x3 stride-1 blocks on a small map in one kernel on 2-CTA clusters
struct ChainTcPlan;
bool chain_tc_supported(int dtype, const StageGeom* g, int n_layers);
int chain_tc_prepare(int dtype, const BlockArgs* layers, int n_layers, const TcLaunchOpts& opts, ChainTcPlan** out);
int chain_tc_launch(ChainTcPlan* cp, cudaStream_t st);
void chain_tc_destroy(ChainTcPlan* cp);
const char* chain_tc_name(ChainTcPlan* cp);
int chain_tc_trace(ChainTcPlan* cp, cudaStream_t st, unsigned long long* out_host, int* rows, int* cols);
// tensor-core stem (fd_stem_tc.cu)
struct StemTcPlan;
bool stem_tc_supported(int dtype, const StageGeom& g);
int stem_tc_prepare(int dtype, const StageGeom& g, const float* w27_dev, const float* scale_dev, const float* bias_dev, void* out,
                    const TcLaunchOpts& opts, StemTcPlan** res);
int stem_tc_launch(StemTcPlan* sp, const void* x, cudaStream_t st);
void stem_tc_destroy(StemTcPlan* sp);
const char* stem_tc_name(StemTcPlan* sp);
// stem + conv1 + conv2 as one kernel (fd_front_tc.cu)
struct FrontTcPlan;
bool front_tc_shape_ok(int dtype, const StageGeom& g0, const StageGeom& g1, const StageGeom& g2);
int front_tc_items(int n, int h, int w);
void front_tc_layout(int cin, int* out);
int front_tc_prepare(int dtype, const StageGeom& g0, const StageGeom& g1, const StageGeom& g2, const float* w27,
                     const float* sc0, const float* bi0, const BlockArgs& a1, const BlockArgs& a2, void* out0,
                     const TcLaunchOpts& opts, FrontTcPlan** res);
int front_tc_launch(FrontTcPlan* fp, const void* x, cudaStream_t st);
void front_tc_destroy(FrontTcPlan* fp);
const char* front_tc_name(FrontTcPlan* fp);
size_t front_tc_param_bytes(FrontTcPlan* fp);
// dense kxk conv on wgmma (fd_conv_tc.cu)
struct ConvTcPlan;
bool conv_tc_supported(int dtype, const StageGeom& g, int kind);
int conv_tc_prepare(int dtype, int kind, const StageGeom& g, const void* in, const void* w, const float* scale_dev,
                    const float* bias_dev, void* out, const TcLaunchOpts& opts, ConvTcPlan** res);
int conv_tc_launch(ConvTcPlan* cp, cudaStream_t st);
void conv_tc_destroy(ConvTcPlan* cp);
const char* conv_tc_name(ConvTcPlan* cp);
// the split-TF32 pointwise step of an fp32 DWPW stage (fd_conv_tc.cu)
bool pw_tf32x3_supported(const StageGeom& g);
bool conv_tc_tf32x3_supported(const StageGeom& g, int kind);
int conv_tc_tf32x3_prepare(int kind, const StageGeom& g, const void* in, const float* w_split, const float* scale_dev,
                           const float* bias_dev, void* out, const TcLaunchOpts& opts, ConvTcPlan** res);
int pw_tf32x3_prepare(const StageGeom& g, const void* mid, const float* w_split, const float* scale_dev, const float* bias_dev,
                      void* out, int out_pitch, int reduce, const TcLaunchOpts& opts, ConvTcPlan** res);
int tf32_split_weights(const float* w, size_t count, float* dst);
// a 16-bit DWPW stage as two steps (fd_conv_tc.cu): the depthwise half into the stage's intermediate, the pointwise half as a
// 1x1 step of conv_tc_kernel; and the plan the block kernel would run the stage with (fd_block_tc.cu)
bool pw_tc_supported(int dtype, const StageGeom& g);
int pw_tc_prepare(int dtype, const StageGeom& g, const void* mid, const void* w, const float* scale_dev, const float* bias_dev,
                  void* out, int out_pitch, int reduce, const TcLaunchOpts& opts, ConvTcPlan** res);
int dw_mid_launch(int dtype, const BlockArgs& a, cudaStream_t st);
BlockPlanOut block_tc_plan_for(const StageGeom& g, const TcLaunchOpts& opts, bool* pinned);
// device memory a kernel plan holds: its packed / padded parameter copies
size_t block_tc_param_bytes(BlockTcPlan* bp);
size_t chain_tc_param_bytes(ChainTcPlan* cp);
size_t stem_tc_param_bytes(StemTcPlan* sp);
size_t conv_tc_param_bytes(ConvTcPlan* cp);

static size_t dtype_size(int dtype) { return dtype == FD_F32 ? 4 : 2; }
static bool is_phased(int kind) { return kind == FD_STAGE_DECONV || kind == FD_STAGE_UPCONV; }
static bool is_conv(int kind) { return kind == FD_STAGE_CONV || is_phased(kind); }

struct Stage {
    fd_stage_desc d{};
    StageGeom g{};
    int out_h = 0, out_w = 0;            // spatial size of the stage's output buffer (after upsample)
    void* out = nullptr;                 // NHWC [n,out_h,out_w,c_out]   (STEM/DWPW)
    void* out_alloc = nullptr;           // what this stage cudaMalloc'ed (out may be a channel slice of another stage's buffer)
    int out_c = 0;                       // channels the NEXT stage sees (c_out, or c_out + c_skip after a concat)
    int out_pitch = 0;                   // elements between pixels of `out`
    int concat_src = -1;                 // >= 0: this stage's output is a channel slice of stage concat_src's wide buffer
    void* mid = nullptr;                 // NHWC [n,h_out,w_out,c_in]     (DWPW, path 0)
    float* dw_w = nullptr;               // [k*k][c_in]
    float* dw_scale = nullptr;
    float* dw_bias = nullptr;
    void* pw_w = nullptr;                // [c_out][c_in] plan dtype (DWPW); [c_out][k*k][c_in] plan dtype (CONV, DECONV, UPCONV)
    float* pw_w_f32 = nullptr;           // stem: [27][c_out] tap-major ; head: [c_in]
    float* pw_scale = nullptr;
    float* pw_bias = nullptr;
    float* w_split = nullptr;            // tf32x3: pw_w split into [2][...] fp32 TF32 high then low parts, shared by every step set
    float head_scale = 0.f, head_bias = 0.f;
    bool have_weights = false;
};

// What one step set built for one stage.
struct StageRun {
    BlockTcPlan* tc = nullptr;
    StemTcPlan* stc = nullptr;
    ConvTcPlan* ctc = nullptr;
    ChainTcPlan* chain = nullptr;        // set on the FIRST stage of a run executed by the chain kernel
    FrontTcPlan* front = nullptr;        // set on the stem when stages 0..2 run as one front_tc_kernel step
    int chained = 0;                     // 1: this stage runs inside a kernel launched at an earlier stage: a chain kernel (its own
                                         //    output buffer is only written if it is the run's last stage) or the front kernel
    void* out_eff = nullptr;             // buffer the stage really writes (== a skip source when accumulating in place)
};

struct Step {
    int stage;
    std::string name;
    double alg_bytes, macs;
    double dw_macs = 0.0;                // of which depthwise (SIMT FMA pipe); the rest is the dense contraction (tensor pipe)
    std::function<int(cudaStream_t, const void*, void*)> run;
};

// The geometry of one stage in a forward of n images at h x w.
struct StageShape {
    StageGeom g{};
    int out_h = 0, out_w = 0;            // spatial size of the stage's output buffer (after upsample)
    int out_c = 0;                       // channels the NEXT stage sees (c_out, or c_out + c_skip after a concat)
};

// The steps of a forward of n images at h x w over the front of the plan's buffers.  Planner choices, grids, item counts
// and tensor maps depend on (n, h, w); the activation buffers, packed weights and split weights are the plan's and shared
// by every set.
struct StepSet {
    int n = 0, h = 0, w = 0;
    std::vector<Step> steps;
    std::vector<StageRun> runs;          // per stage
    size_t bytes = 0;                    // device memory its kernel plans hold (packed parameter copies)
    unsigned long long stamp = 0;
};

}  // namespace fd

using namespace fd;

struct fd_plan {
    int n = 0, h = 0, w = 0, dtype = 0, device = 0, n_sms = 132;
    std::vector<Stage> stages;
    std::vector<StepSet*> sets;          // built lazily per live (n, h, w); LRU-bounded, the set of the plan's own (N, H, W) is kept
    unsigned long long set_clock = 0;
    int opt_path = 1, opt_fold_head = 1, opt_graph = 1, opt_tma_epilogue = 1, opt_inplace_skip = 1, opt_pdl = 0, opt_wait_sleep_ns = 0;
    int opt_chain = 1;
    int opt_cluster = 1;
    int opt_tf32x3 = 0;
    int opt_unfuse = 1;
    int opt_front = 1;
    size_t workspace_bytes = 0;
    size_t split_bytes = 0;              // device memory of the stages' split weights (tf32x3), freed with the step sets
    // fd_pipeline_*: host batches flow H2D -> forward -> D2H through kPipeSlots device slots on three streams
    struct PipeSlot { void* x = nullptr; void* y = nullptr; cudaEvent_t up = nullptr, done = nullptr, down = nullptr; bool busy = false; };
    PipeSlot pipe[3];
    cudaStream_t pipe_h2d = nullptr, pipe_run = nullptr, pipe_d2h = nullptr;
    unsigned long long pipe_next = 0;    // next ticket
    void* stage_x = nullptr;             // device staging for fd_forward_host
    void* stage_y = nullptr;
    cudaEvent_t last_done = nullptr;     // recorded after every fd_forward on its stream (cross-stream ordering of one plan's buffers)
    cudaStream_t last_stream = nullptr;
    bool last_stream_set = false;
    void* l2_flush = nullptr;
    size_t l2_flush_bytes = 0;
    // CUDA graph cache keyed on the (x, y) pointer pair and the shape (n, h, w): callers that rotate a few buffers (or let a
    // caching allocator hand the same blocks back, possibly for another shape) replay; a new key is captured once, LRU-evicted.
    struct GraphEntry { const void* x; void* y; int n, h, w; cudaGraphExec_t exec; unsigned long long stamp; };
    std::vector<GraphEntry> graphs;
    unsigned long long graph_clock = 0;
    int graph_misses = 0;                // consecutive fd_forward calls that found no captured graph for their (x, y) pair
};
static const size_t kMaxGraphs = 8;
// the automatic two-step route is for stages whose depthwise intermediate stays in the 50 MB L2 between its two steps
static const size_t kUnfuseMaxMidBytes = size_t(16) << 20;
static const size_t kMaxStepSets = 8;

namespace fd {

struct DeviceGuard {
    int prev = -1;
    bool ok = true;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) { ok = false; return; }
        if (prev != dev && cudaSetDevice(dev) != cudaSuccess) ok = false;
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

static int dev_alloc(fd_plan* p, void** ptr, size_t bytes) {
    bytes = (bytes + 255) & ~size_t(255);
    FD_CUDA_OK(cudaMalloc(ptr, bytes));
    FD_CUDA_OK(cudaMemset(*ptr, 0, bytes));
    // the fill runs on the legacy default stream, which the plan's non-blocking pipeline streams do not wait for: let it
    // finish before one of them uploads into the buffer
    FD_CUDA_OK(cudaStreamSynchronize(cudaStreamLegacy));
    p->workspace_bytes += bytes;
    return FD_OK;
}

static void destroy_set(StepSet* ss) {
    for (auto& r : ss->runs) {
        if (r.tc) block_tc_destroy(r.tc);
        if (r.stc) stem_tc_destroy(r.stc);
        if (r.ctc) conv_tc_destroy(r.ctc);
        if (r.chain) chain_tc_destroy(r.chain);
        if (r.front) front_tc_destroy(r.front);
    }
    delete ss;
}

static StepSet* find_set(fd_plan* p, int n, int h, int w) {
    for (StepSet* ss : p->sets)
        if (ss->n == n && ss->h == h && ss->w == w) return ss;
    return nullptr;
}

// the set of the plan's own (N, H, W): never evicted, and the one the introspection functions describe
static bool is_capacity_set(const fd_plan* p, const StepSet* ss) { return ss->n == p->n && ss->h == p->h && ss->w == p->w; }

// weights or options changed: every step set, every graph and the split weights go
static void invalidate(fd_plan* p) {
    for (auto& g : p->graphs) cudaGraphExecDestroy(g.exec);
    p->graphs.clear();
    for (StepSet* ss : p->sets) destroy_set(ss);
    p->sets.clear();
    for (auto& s : p->stages) { cudaFree(s.w_split); s.w_split = nullptr; }
    p->split_bytes = 0;
}

// the stage's pw_w ([c_out][k*k][c_in], fp32) split once into its TF32 high and low parts, for every step set
static int split_weights(fd_plan* p, Stage& s, size_t count, const float** out) {
    if (!s.w_split) {
        FD_CUDA_OK(cudaMalloc(&s.w_split, 2 * count * sizeof(float)));
        int rc = tf32_split_weights(static_cast<const float*>(s.pw_w), count, s.w_split);
        if (rc != FD_OK) { cudaFree(s.w_split); s.w_split = nullptr; return rc; }
        p->split_bytes += 2 * count * sizeof(float);
    }
    *out = s.w_split;
    return FD_OK;
}

// fp32 host array -> device array of the plan dtype (exact when the values came from that dtype)
static int upload_as_dtype(int dtype, const float* host, size_t count, void* dev) {
    if (dtype == FD_F32) {
        FD_CUDA_OK(cudaMemcpy(dev, host, count * 4, cudaMemcpyHostToDevice));
    } else if (dtype == FD_F16) {
        std::vector<__half> tmp(count);
        for (size_t i = 0; i < count; ++i) tmp[i] = __float2half_rn(host[i]);
        FD_CUDA_OK(cudaMemcpy(dev, tmp.data(), count * 2, cudaMemcpyHostToDevice));
    } else {
        std::vector<__nv_bfloat16> tmp(count);
        for (size_t i = 0; i < count; ++i) tmp[i] = __float2bfloat16_rn(host[i]);
        FD_CUDA_OK(cudaMemcpy(dev, tmp.data(), count * 2, cudaMemcpyHostToDevice));
    }
    return FD_OK;
}

// Walk the stage list for a forward of n images at h x w: check every stage against its producer and return each stage's
// geometry.  fd_plan_create sizes the plan's buffers from the walk at (N, H, W); every step set repeats it at its own shape.
static int walk_stages(const fd_stage_desc* stages, int n_stages, int n, int h, int w, std::vector<StageShape>& out) {
    out.assign(n_stages, StageShape());
    std::vector<int> concat_src(n_stages, -1);         // >= 0: the stage's output is a channel slice of that stage's buffer
    // the stem reads c_in planes of x: 1..7 (RGB 3, depth only 1, RGB-D 4; K = 9 c_in fits one 64-element row of the
    // tensor-core stem).  8 or more would need a second K block per im2col row
    const int c_x = stages[0].c_in;
    if (stages[0].kind == FD_STAGE_STEM && c_x <= 0) return fail(FD_ERR_INVALID, "stem c_in must be positive");
    if (stages[0].kind == FD_STAGE_STEM && c_x > 7)
        return fail(FD_ERR_UNSUPPORTED, "stem c_in " + std::to_string(c_x) + " is not supported: the stem takes 1..7 input channels");
    int ch = c_x, hh = h, ww = w;
    for (int i = 0; i < n_stages; ++i) {
        const fd_stage_desc& d = stages[i];
        StageShape& s = out[i];
        const bool first = i == 0, lastst = i == n_stages - 1;
        if ((d.kind == FD_STAGE_STEM) != first || (d.kind == FD_STAGE_HEAD) != lastst ||
            (!first && !lastst && d.kind != FD_STAGE_DWPW && !is_conv(d.kind)))
            return fail(FD_ERR_INVALID, "stage list must be STEM, (DWPW|CONV|DECONV|UPCONV)..., HEAD");
        if (d.c_in != ch) return fail(FD_ERR_INVALID, "stage " + std::to_string(i) + ": c_in does not match producer");
        if (d.act != FD_ACT_RELU && d.act != FD_ACT_RELU6) return fail(FD_ERR_INVALID, "bad act");
        s.g.n = n; s.g.h_in = hh; s.g.w_in = ww; s.g.c_in = d.c_in; s.g.c_out = d.c_out;
        s.g.ksize = d.ksize; s.g.stride = d.stride; s.g.act = d.act; s.g.upsample = d.upsample ? 1 : 0;
        if (d.kind == FD_STAGE_STEM) {
            if (d.ksize != 3 || d.c_out % 8 || d.stride < 1 || d.stride > 2 || d.upsample || d.skip_src >= 0)
                return fail(FD_ERR_INVALID, "stem must be 3x3, c_out % 8 == 0, stride 1|2");
            s.g.h_out = (hh + 2 - 3) / d.stride + 1; s.g.w_out = (ww + 2 - 3) / d.stride + 1;
        } else if (d.kind == FD_STAGE_DWPW) {
            if ((d.ksize != 3 && d.ksize != 5) || d.stride < 1 || d.stride > 2 || d.c_in % 8 || d.c_out % 8 || d.c_out <= 0)
                return fail(FD_ERR_INVALID, "block stage needs k in {3,5}, stride 1|2, channels % 8 == 0");
            const int pad = (d.ksize - 1) / 2;
            s.g.h_out = (hh + 2 * pad - d.ksize) / d.stride + 1; s.g.w_out = (ww + 2 * pad - d.ksize) / d.stride + 1;
        } else if (d.kind == FD_STAGE_CONV) {
            if (d.skip_src >= 0) return fail(FD_ERR_INVALID, "stage " + std::to_string(i) + ": a CONV stage takes no skip");
            if (d.stride != 1) return fail(FD_ERR_INVALID, "stage " + std::to_string(i) + ": a CONV stage has stride 1");
            if ((d.ksize != 3 && d.ksize != 5) || d.c_in % 8 || d.c_out % 8 || d.c_out <= 0 || (d.upsample != 0 && d.upsample != 1))
                return fail(FD_ERR_INVALID, "conv stage needs k in {3,5}, channels % 8 == 0, upsample 0|1");
            s.g.h_out = hh; s.g.w_out = ww;
        } else if (is_phased(d.kind)) {
            const char* nm = d.kind == FD_STAGE_DECONV ? "a DECONV" : "an UPCONV";
            if (d.skip_src >= 0) return fail(FD_ERR_INVALID, "stage " + std::to_string(i) + ": " + nm + " stage takes no skip");
            if (d.stride != 2) return fail(FD_ERR_INVALID, "stage " + std::to_string(i) + ": " + nm + " stage has stride 2");
            if (d.upsample != 0) return fail(FD_ERR_INVALID, "stage " + std::to_string(i) + ": " + nm + " stage has upsample 0");
            const bool k_ok = d.kind == FD_STAGE_DECONV ? (d.ksize == 3 || d.ksize == 5 || d.ksize == 7 || d.ksize == 9) : d.ksize == 5;
            if (!k_ok || d.c_in % 8 || d.c_out % 8 || d.c_out <= 0)
                return fail(FD_ERR_INVALID, d.kind == FD_STAGE_DECONV ? "deconv stage needs k in {3,5,7,9}, channels % 8 == 0"
                                                                      : "upconv stage needs k 5, channels % 8 == 0");
            s.g.h_out = hh; s.g.w_out = ww;            // the phase convs run at the input resolution; the output is 2h x 2w
        } else {
            if (d.ksize != 1 || d.c_out != 1 || d.c_in % 8 || d.upsample || d.skip_src >= 0)
                return fail(FD_ERR_INVALID, "head must be 1x1, c_out 1, c_in % 8 == 0");
            s.g.h_out = hh; s.g.w_out = ww;
        }
        s.out_h = s.g.h_out * (s.g.upsample || is_phased(d.kind) ? 2 : 1);
        s.out_w = s.g.w_out * (s.g.upsample || is_phased(d.kind) ? 2 : 1);
        s.out_c = d.c_out;
        if (d.skip_src >= 0) {
            if (d.kind != FD_STAGE_DWPW || !d.upsample || d.skip_src >= i) return fail(FD_ERR_INVALID, "bad skip_src");
            const StageShape& src = out[d.skip_src];
            if (src.out_h != s.out_h || src.out_w != s.out_w || (!d.skip_mode && src.g.c_out != d.c_out))
                return fail(FD_ERR_INVALID, "stage " + std::to_string(i) + ": skip tensor shape does not match the upsampled output");
            if (d.skip_mode) {
                // concatenation (models.py:806-811): the stage's output is one wide NHWC buffer [.., c_out + c_skip]
                if (d.skip_mode != 1 || concat_src[d.skip_src] >= 0 || stages[d.skip_src].skip_src >= 0)
                    return fail(FD_ERR_INVALID, "bad skip_mode / skip source");
                s.out_c = d.c_out + src.g.c_out;
                concat_src[d.skip_src] = i;
            }
        }
        ch = s.out_c; hh = s.out_h; ww = s.out_w;
    }
    if (hh != h || ww != w) return fail(FD_ERR_INVALID, "stage list does not return to the input resolution");
    return FD_OK;
}

// The front route (plan option "front"): the stem and the two DWPW stages after it run as one front_tc_kernel step when the
// three have the stock MobileNet shapes (front_tc_shape_ok), neither block takes a skip or upsamples, and no stage
// concatenates onto one of their outputs (a channel slice of a wider buffer).  A 16-bit plan on path 1 only.
static bool front_route_ok(const fd_stage_desc* D, int ns, int dtype, const std::vector<StageShape>& S) {
    if (ns < 4 || D[0].kind != FD_STAGE_STEM || D[1].kind != FD_STAGE_DWPW || D[2].kind != FD_STAGE_DWPW) return false;
    if (D[1].skip_src >= 0 || D[2].skip_src >= 0) return false;
    for (int j = 3; j < ns; ++j)
        if (D[j].skip_src >= 0 && D[j].skip_src <= 2 && D[j].skip_mode) return false;
    return front_tc_shape_ok(dtype, S[0].g, S[1].g, S[2].g);
}

// Build the steps of a forward of n images at h x w into `ss`: every stage's geometry at that shape, over the front of the
// plan's buffers.  Every decision that depends on the geometry (the chain kernel, the two-step route, the planners) is
// taken from the set's own geometry, as a plan built for (n, h, w) takes it.
static int build_steps(fd_plan* p, int n, int h, int w, StepSet* ss) {
    const int ns = (int)p->stages.size();
    const double es = (double)dtype_size(p->dtype);
    for (auto& s : p->stages)
        if (!s.have_weights) return fail(FD_ERR_STATE, "fd_plan_set_stage_weights was not called for every stage");
    ss->n = n; ss->h = h; ss->w = w;
    ss->runs.assign(ns, StageRun());
    std::vector<StageRun>& R = ss->runs;
    std::vector<fd_stage_desc> D(ns);
    for (int i = 0; i < ns; ++i) D[i] = p->stages[i].d;
    std::vector<StageShape> S;
    int wrc = walk_stages(D.data(), ns, n, h, w, S);
    if (wrc != FD_OK) return wrc;
    std::vector<StageGeom> G(ns);
    for (int i = 0; i < ns; ++i) G[i] = S[i].g;

    TcLaunchOpts lopts;                   // every kernel plan keeps its own copy (no process-wide launch state)
    lopts.pdl = p->opt_pdl; lopts.sleep_ns = p->opt_wait_sleep_ns; lopts.n_sms = p->n_sms; lopts.cluster = p->opt_cluster;
    Stage& head = p->stages[ns - 1];
    Stage& last = p->stages[ns - 2];
    // decode_conv6 below the last upsample: exact because a 1x1 conv, a per-channel affine and ReLU
    // act pixel-wise and nearest upsampling only replicates pixels (SURVEY.md section 2b row 8).
    const bool fold = p->opt_fold_head && (last.d.kind == FD_STAGE_DWPW || last.d.kind == FD_STAGE_CONV) && last.d.upsample &&
                      last.d.skip_src < 0;
    bool head_fused = false;

    for (int i = 0; i < ns; ++i) {
        Stage& s = p->stages[i];
        StageRun& r = R[i];
        StageGeom& sg = G[i];
        const void* in = i > 0 ? R[i - 1].out_eff : nullptr;
        r.out_eff = s.out;
        sg.in_pitch = i > 0 ? p->stages[i - 1].out_pitch : 0;
        sg.out_pitch = s.out_pitch;
        sg.skip_pitch = (s.d.skip_src >= 0 && !s.d.skip_mode) ? p->stages[s.d.skip_src].out_pitch : s.out_pitch;
        if (s.d.kind == FD_STAGE_STEM) {
            Step st;
            st.stage = i;
            st.name = sg.c_in == 3 ? "stem_kernel" : "stem_kernel<cin" + std::to_string(sg.c_in) + ">";
            st.macs = (double)sg.n * sg.h_out * sg.w_out * sg.c_out * 9.0 * sg.c_in;
            st.alg_bytes = ((double)sg.n * sg.c_in * sg.h_in * sg.w_in + (double)sg.n * sg.h_out * sg.w_out * sg.c_out) * es +
                           (9.0 * sg.c_in + 2.0) * sg.c_out * 4;
            Stage* sp = &s;
            const int dtype = p->dtype;
            if (p->opt_path == 1 && p->opt_front && front_route_ok(D.data(), ns, dtype, S) && stem_tc_supported(dtype, sg)) {
                // stem + conv1 + conv2 as one step that writes all three buffers and reads only x; reported under stage 2,
                // the last buffer it writes, as a chain run is
                BlockArgs a[2]{};
                StageGeom g[3] = {sg, G[1], G[2]};
                for (int k = 1; k <= 2; ++k) {
                    Stage& t = p->stages[k];
                    g[k].in_pitch = p->stages[k - 1].out_pitch; g[k].out_pitch = t.out_pitch;
                    BlockArgs& b = a[k - 1];
                    b.g = g[k]; b.out = t.out;
                    b.dw_w = t.dw_w; b.dw_scale = t.dw_scale; b.dw_bias = t.dw_bias;
                    b.pw_w = t.pw_w; b.pw_scale = t.pw_scale; b.pw_bias = t.pw_bias;
                }
                int rc = front_tc_prepare(dtype, g[0], g[1], g[2], s.pw_w_f32, s.pw_scale, s.pw_bias, a[0], a[1], s.out, lopts, &r.front);
                if (rc != FD_OK) return rc;
                ss->bytes += front_tc_param_bytes(r.front);
                st.stage = 2;
                st.name = front_tc_name(r.front);
                st.dw_macs = 0.0;
                double wb = (9.0 * sg.c_in + 2.0) * sg.c_out * 4, out_px_bytes = (double)sg.n * sg.h_out * sg.w_out * sg.c_out;
                for (int k = 1; k <= 2; ++k) {
                    const double px = (double)g[k].n * g[k].h_out * g[k].w_out;
                    st.dw_macs += px * g[k].c_in * 9.0;
                    st.macs += px * g[k].c_in * 9.0 + px * g[k].c_in * g[k].c_out;
                    wb += (double)g[k].c_in * 9 * 4 + 2.0 * g[k].c_in * 4 + (double)g[k].c_in * g[k].c_out * es + 2.0 * g[k].c_out * 4;
                    out_px_bytes += px * g[k].c_out;
                    R[k].chained = 1;
                    R[k].out_eff = p->stages[k].out;
                }
                st.alg_bytes = ((double)sg.n * sg.c_in * sg.h_in * sg.w_in + out_px_bytes) * es + wb;
                FrontTcPlan* fp = r.front;
                st.run = [fp](cudaStream_t stream, const void* x, void*) { return front_tc_launch(fp, x, stream); };
            } else if (p->opt_path == 1 && stem_tc_supported(dtype, sg)) {
                int rc = stem_tc_prepare(dtype, sg, s.pw_w_f32, s.pw_scale, s.pw_bias, s.out, lopts, &r.stc);
                if (rc != FD_OK) return rc;
                ss->bytes += stem_tc_param_bytes(r.stc);
                st.name = stem_tc_name(r.stc);
                StemTcPlan* stc = r.stc;
                st.run = [stc](cudaStream_t stream, const void* x, void*) { return stem_tc_launch(stc, x, stream); };
            } else {
                const StageGeom g = sg;
                st.run = [sp, dtype, g](cudaStream_t stream, const void* x, void*) {
                    return launch_stem(dtype, x, sp->out, sp->pw_w_f32, sp->pw_scale, sp->pw_bias, g, stream);
                };
            }
            ss->steps.push_back(st);
        } else if (is_conv(s.d.kind)) {
            // dense kxk conv: one implicit-GEMM step (path 1: conv_tc_kernel, else the SIMT conv_kernel); with the head folded
            // below the last upsample the stage stores at conv resolution and head_kernel<up2x> replicates.  DECONV / UPCONV:
            // the same step as four phase convs at the input resolution (g.h_out == g.h_in), k*k*c_in*c_out MACs per input
            // pixel, the 2h x 2w output written once (path 0: convt_kernel)
            StageGeom g = sg;
            if (fold && &s == &last) g.upsample = 0;
            const int kind = s.d.kind;
            const double px_in = (double)g.n * g.h_in * g.w_in, px_out = (double)g.n * g.h_out * g.w_out;
            const double kk = (double)g.ksize * g.ksize;
            Step st;
            st.stage = i;
            st.macs = px_out * g.c_in * g.c_out * kk;
            st.dw_macs = 0.0;
            st.alg_bytes = (px_in * g.c_in + px_out * (g.upsample || is_phased(kind) ? 4.0 : 1.0) * g.c_out) * es +
                           kk * g.c_in * g.c_out * es + 2.0 * g.c_out * 4;
            const int dtype = p->dtype;
            if (dtype == FD_F32 && p->opt_path == 1 && p->opt_tf32x3 && conv_tc_tf32x3_supported(g, kind)) {
                // fp32 under tf32x3: the same implicit GEMM as split TF32 (conv_tc_tf32x3_kernel), three TF32 products per
                // term; the weights are split once into their TF32 high and low parts, a buffer twice the fp32 weights
                const float* w_split = nullptr;
                int rc = split_weights(p, s, (size_t)g.c_out * g.ksize * g.ksize * g.c_in, &w_split);
                if (rc != FD_OK) return rc;
                rc = conv_tc_tf32x3_prepare(kind, g, in, w_split, s.pw_scale, s.pw_bias, s.out, lopts, &r.ctc);
                if (rc != FD_OK) return rc;
                ss->bytes += conv_tc_param_bytes(r.ctc);
                st.name = conv_tc_name(r.ctc);
                ConvTcPlan* ctc = r.ctc;
                st.run = [ctc](cudaStream_t stream, const void*, void*) { return conv_tc_launch(ctc, stream); };
            } else if (p->opt_path == 1 && conv_tc_supported(dtype, g, kind)) {
                int rc = conv_tc_prepare(dtype, kind, g, in, s.pw_w, s.pw_scale, s.pw_bias, s.out, lopts, &r.ctc);
                if (rc != FD_OK) return rc;
                ss->bytes += conv_tc_param_bytes(r.ctc);
                st.name = conv_tc_name(r.ctc);
                ConvTcPlan* ctc = r.ctc;
                st.run = [ctc](cudaStream_t stream, const void*, void*) { return conv_tc_launch(ctc, stream); };
            } else if (kind == FD_STAGE_CONV) {
                char nm[64];
                snprintf(nm, sizeof(nm), "conv_kernel<k%d>", g.ksize);
                st.name = nm;
                Stage* sp = &s;
                st.run = [sp, in, g, dtype](cudaStream_t stream, const void*, void*) {
                    return launch_conv(dtype, in, sp->pw_w, sp->out, sp->pw_scale, sp->pw_bias, g, stream);
                };
            } else {
                char nm[64];
                snprintf(nm, sizeof(nm), "convt_kernel<%s%d>", kind == FD_STAGE_DECONV ? "deconv" : "upconv", g.ksize);
                st.name = nm;
                Stage* sp = &s;
                st.run = [sp, in, g, dtype, kind](cudaStream_t stream, const void*, void*) {
                    return launch_convt(dtype, kind, in, sp->pw_w, sp->out, sp->pw_scale, sp->pw_bias, g, stream);
                };
            }
            ss->steps.push_back(st);
        } else if (s.d.kind == FD_STAGE_DWPW && r.chained) {
            continue;                                 // executed by the chain kernel launched at the run's first stage
        } else if (s.d.kind == FD_STAGE_DWPW) {
            // ---- a run of 3x3 stride-1 blocks on a small map: ONE chain kernel (2-CTA clusters, activations stay in shared memory)
            if (p->opt_path == 1 && p->opt_chain) {
                std::vector<BlockArgs> run;
                std::vector<StageGeom> geoms;
                int j = i;
                for (; j < ns - 1 && (int)run.size() < 8; ++j) {
                    Stage& t = p->stages[j];
                    if (t.d.kind != FD_STAGE_DWPW || t.d.ksize != 3 || t.d.stride != 1 || t.d.upsample || t.d.skip_src >= 0) break;
                    if (j > i && p->stages[j - 1].concat_src >= 0) break;     // the previous output must really be written (concat slice)
                    bool is_skip_source = false;                              // ... and so must a tensor a decoder stage will add / concatenate
                    for (int k2 = j + 1; k2 < ns; ++k2) if (p->stages[k2].d.skip_src == j) is_skip_source = true;
                    BlockArgs b{};
                    b.g = G[j];
                    b.g.in_pitch = j > 0 ? p->stages[j - 1].out_pitch : 0;
                    b.g.out_pitch = t.out_pitch;
                    b.in = j > 0 ? R[j - 1].out_eff : nullptr;
                    b.out = t.out;
                    b.dw_w = t.dw_w; b.dw_scale = t.dw_scale; b.dw_bias = t.dw_bias;
                    b.pw_w = t.pw_w; b.pw_scale = t.pw_scale; b.pw_bias = t.pw_bias;
                    run.push_back(b); geoms.push_back(b.g);
                    if (is_skip_source) { ++j; break; }                       // a skip source may END a run, not sit inside one
                }
                int len = (int)run.size();
                while (len >= 2 && !chain_tc_supported(p->dtype, geoms.data(), len)) --len;
                if (len >= 2) {
                    int rc = chain_tc_prepare(p->dtype, run.data(), len, lopts, &r.chain);
                    if (rc != FD_OK) return rc;
                    ss->bytes += chain_tc_param_bytes(r.chain);
                    Step st;
                    st.stage = i + len - 1;                                   // reported under the run's last stage (the tensor it writes)
                    st.macs = 0; st.dw_macs = 0;
                    double wb = 0;
                    for (int k2 = 0; k2 < len; ++k2) {
                        const StageGeom& g = geoms[k2];
                        const double px = (double)g.n * g.h_out * g.w_out;
                        st.dw_macs += px * g.c_in * 9.0;
                        st.macs += px * g.c_in * 9.0 + px * g.c_in * g.c_out;
                        wb += (double)g.c_in * 9 * 4 + 2.0 * g.c_in * 4 + (double)g.c_in * g.c_out * es + 2.0 * g.c_out * 4;
                        R[i + k2].chained = 1;
                        R[i + k2].out_eff = p->stages[i + k2].out;
                    }
                    // algorithmic bytes of the MERGED stage (SURVEY.md 8d rule): external input once + external output once + weights once
                    st.alg_bytes = ((double)geoms[0].n * geoms[0].h_in * geoms[0].w_in * geoms[0].c_in +
                                    (double)geoms[len - 1].n * geoms[len - 1].h_out * geoms[len - 1].w_out * geoms[len - 1].c_out) * es + wb;
                    char nm[200];
                    snprintf(nm, sizeof(nm), "%s{stages %d-%d}", chain_tc_name(r.chain), i, i + len - 1);
                    st.name = nm;
                    ChainTcPlan* cpn = r.chain;
                    st.run = [cpn](cudaStream_t stream, const void*, void*) { return chain_tc_launch(cpn, stream); };
                    ss->steps.push_back(st);
                    r.chained = 1;
                    continue;
                }
            }
            BlockArgs a{};
            a.g = sg;
            const bool folded_here = fold && (&s == &last);
            if (folded_here) a.g.upsample = 0;
            a.in = in;
            a.mid = s.mid;
            a.out = s.out;
            a.skip = (s.d.skip_src >= 0 && !s.d.skip_mode) ? R[s.d.skip_src].out_eff : nullptr;   // concat: the source wrote its slice itself
            a.dw_w = s.dw_w; a.dw_scale = s.dw_scale; a.dw_bias = s.dw_bias;
            a.pw_w = s.pw_w; a.pw_scale = s.pw_scale; a.pw_bias = s.pw_bias;
            const double px_in = (double)sg.n * sg.h_in * sg.w_in, px_out = (double)sg.n * sg.h_out * sg.w_out;
            const double up = a.g.upsample ? 4.0 : 1.0;
            const double dw_macs = px_out * sg.c_in * sg.ksize * sg.ksize, pw_macs = px_out * sg.c_in * sg.c_out;
            const double w_bytes = (double)sg.c_in * sg.ksize * sg.ksize * 4 + 2.0 * sg.c_in * 4 +
                                   (double)sg.c_in * sg.c_out * es + 2.0 * sg.c_out * 4;
            const double fused_bytes = (px_in * sg.c_in + px_out * up * sg.c_out * (a.skip ? 2.0 : 1.0)) * es + w_bytes;
            const int dtype = p->dtype;
            const bool fuse_head = folded_here && p->opt_path == 1 && block_tc_supported(dtype, a.g, true);
            bool use_tc = p->opt_path == 1 && block_tc_supported(dtype, a.g, false);
            // ---- the two-step route (plan option "unfuse"): the depthwise half once into `mid`, then the pointwise half as a
            // 1x1 step of conv_tc_kernel.  The block kernel holds an item's accumulator in registers, 128 output channels at
            // most, and every output-channel split recomputes the depthwise half and reloads the halo tile; where it would
            // split 8 ways or more, or hand the operand tiles around a tile-sharing cluster, the stage's map is small enough
            // to stay in the L2 between the two steps and fusion costs more than it saves.  Same bits either way.
            const bool add_in_place = a.skip != nullptr && p->opt_tma_epilogue && p->opt_inplace_skip;
            if (use_tc && p->opt_unfuse && !folded_here && (a.skip == nullptr || add_in_place) && pw_tc_supported(dtype, a.g)) {
                bool pinned = false;
                const BlockPlanOut bpo = block_tc_plan_for(a.g, lopts, &pinned);
                const size_t mid_bytes = (size_t)px_out * sg.c_in * dtype_size(dtype);
                const bool wide = bpo.ok && (bpo.splits >= 8 || bpo.cs > 1) && mid_bytes <= kUnfuseMaxMidBytes;
                if (!pinned && (p->opt_unfuse == 2 || wide)) {
                    void* out = a.skip ? const_cast<void*>(a.skip) : a.out;         // a skip is added where it lies
                    const int opitch = a.skip ? a.g.skip_pitch : a.g.out_pitch;
                    if (a.skip) r.out_eff = out;
                    int rc = pw_tc_prepare(dtype, a.g, a.mid, a.pw_w, a.pw_scale, a.pw_bias, out, opitch, a.skip ? 1 : 0, lopts, &r.ctc);
                    if (rc != FD_OK) return rc;
                    ss->bytes += conv_tc_param_bytes(r.ctc);
                    Step d;
                    d.stage = i;
                    d.name = sg.ksize == 3 ? "dw_mid_kernel<3>" : "dw_mid_kernel<5>";
                    d.macs = dw_macs;
                    d.dw_macs = dw_macs;
                    d.alg_bytes = (px_in + px_out) * sg.c_in * es + (double)sg.c_in * (sg.ksize * sg.ksize + 2) * 4;
                    d.run = [a, dtype](cudaStream_t stream, const void*, void*) { return dw_mid_launch(dtype, a, stream); };
                    ss->steps.push_back(d);
                    Step q;
                    q.stage = i;
                    q.name = std::string("pw:") + conv_tc_name(r.ctc);      // the pointwise half of a DWPW stage, not a CONV stage
                    q.macs = pw_macs;
                    q.alg_bytes = (px_out * sg.c_in + px_out * up * sg.c_out * (a.skip ? 2.0 : 1.0)) * es +
                                  (double)sg.c_in * sg.c_out * es + 2.0 * sg.c_out * 4;
                    ConvTcPlan* ctc = r.ctc;
                    q.run = [ctc](cudaStream_t stream, const void*, void*) { return conv_tc_launch(ctc, stream); };
                    ss->steps.push_back(q);
                    continue;
                }
            }
            if (use_tc) {
                // decoder blocks with a skip accumulate INTO the skip tensor (TMA reduce-add): that buffer becomes the
                // block's output and the skip never has to be read by the SM
                const bool tma_epi = p->opt_tma_epilogue != 0;
                if (tma_epi && p->opt_inplace_skip && a.skip != nullptr) { a.out = const_cast<void*>(a.skip); r.out_eff = a.out; }
                int rc = fuse_head ? block_tc_prepare(dtype, a, head.pw_w_f32, head.head_scale, head.head_bias, G[ns - 1].act, nullptr, false, lopts, &r.tc)
                                   : block_tc_prepare(dtype, a, nullptr, 0.f, 0.f, 0, nullptr, tma_epi && (a.skip == nullptr || a.skip == a.out), lopts, &r.tc);
                if (rc != FD_OK) return rc;
                ss->bytes += block_tc_param_bytes(r.tc);
                Step st;
                st.stage = i;
                st.name = block_tc_name(r.tc);
                st.macs = dw_macs + pw_macs + (fuse_head ? px_out * sg.c_out : 0.0);
                st.dw_macs = dw_macs;
                st.alg_bytes = fuse_head ? (px_in * sg.c_in + px_out * 4.0) * es + w_bytes + sg.c_out * 4.0 : fused_bytes;
                BlockTcPlan* tc = r.tc;
                st.run = [tc](cudaStream_t stream, const void*, void* y) { return block_tc_launch(tc, stream, y); };
                ss->steps.push_back(st);
                head_fused = fuse_head;
            } else {
                Step d;
                d.stage = i;
                d.name = sg.ksize == 3 ? "dw_kernel<3>" : "dw_kernel<5>";
                d.macs = dw_macs;
                d.dw_macs = dw_macs;
                d.alg_bytes = (px_in + px_out) * sg.c_in * es + (double)sg.c_in * (sg.ksize * sg.ksize + 2) * 4;
                d.run = [a, dtype](cudaStream_t stream, const void*, void*) { return launch_dw(dtype, a, stream); };
                ss->steps.push_back(d);
                Step q;
                q.stage = i;
                q.name = "pw_kernel";
                q.macs = pw_macs;
                q.alg_bytes = (px_out * sg.c_in + px_out * up * sg.c_out * (a.skip ? 2.0 : 1.0)) * es +
                              (double)sg.c_in * sg.c_out * es + 2.0 * sg.c_out * 4;
                if (dtype == FD_F32 && p->opt_path == 1 && p->opt_tf32x3 && pw_tf32x3_supported(a.g)) {
                    // the pointwise half as split TF32 on wgmma (conv_tc_tf32x3_kernel).  A skip is added by a TMA reduce-add
                    // of the tiles: into the skip tensor itself (inplace_skip, which then becomes the stage output), or into
                    // the stage's own buffer after a device copy of the skip; either way the result is skip + up rounded once
                    const bool add = a.skip != nullptr;
                    const bool inplace = add && p->opt_inplace_skip;
                    void* out = inplace ? const_cast<void*>(a.skip) : a.out;
                    const int opitch = inplace ? a.g.skip_pitch : a.g.out_pitch;
                    if (inplace) r.out_eff = out;
                    const float* w_split = nullptr;
                    int rc = split_weights(p, s, (size_t)a.g.c_out * a.g.c_in, &w_split);
                    if (rc != FD_OK) return rc;
                    rc = pw_tf32x3_prepare(a.g, a.mid, w_split, a.pw_scale, a.pw_bias, out, opitch, add ? 1 : 0, lopts, &r.ctc);
                    if (rc != FD_OK) return rc;
                    ss->bytes += conv_tc_param_bytes(r.ctc);
                    q.name = conv_tc_name(r.ctc);
                    ConvTcPlan* ctc = r.ctc;
                    const bool copy = add && !inplace;
                    const void* skip = a.skip;
                    const size_t rows = (size_t)a.g.n * S[i].out_h * S[i].out_w, row_bytes = (size_t)a.g.c_out * 4;
                    const size_t dpitch = (size_t)a.g.out_pitch * 4, spitch = (size_t)a.g.skip_pitch * 4;
                    q.run = [ctc, copy, out, skip, rows, row_bytes, dpitch, spitch](cudaStream_t stream, const void*, void*) {
                        if (copy)
                            FD_CUDA_OK(cudaMemcpy2DAsync(out, dpitch, skip, spitch, row_bytes, rows, cudaMemcpyDeviceToDevice, stream));
                        return conv_tc_launch(ctc, stream);
                    };
                } else {
                    q.run = [a, dtype](cudaStream_t stream, const void*, void*) { return launch_pw(dtype, a, stream); };
                }
                ss->steps.push_back(q);
            }
        } else if (!head_fused) {  // HEAD (unless decode_conv6 already ran inside the last block's epilogue)
            const bool up = fold;
            const int hh = up ? G[ns - 2].h_out : sg.h_in, ww = up ? G[ns - 2].w_out : sg.w_in;
            const long long m_total = (long long)sg.n * hh * ww;
            Step st;
            st.stage = i;
            st.name = up ? "head_kernel<up2x>" : "head_kernel";
            st.macs = (double)m_total * sg.c_in;
            st.alg_bytes = ((double)m_total * sg.c_in + (double)sg.n * sg.h_in * sg.w_in) * es + sg.c_in * 4.0;
            Stage* sp = &s;
            const int dtype = p->dtype;
            const int c = sg.c_in, act = sg.act, ipitch = sg.in_pitch;
            st.run = [sp, in, dtype, m_total, c, ipitch, hh, ww, up, act](cudaStream_t stream, const void*, void* y) {
                return launch_head(dtype, in, y, sp->pw_w_f32, sp->head_scale, sp->head_bias, m_total, c, ipitch, hh, ww, up ? 1 : 0,
                                   act, stream);
            };
            ss->steps.push_back(st);
        }
    }
    return FD_OK;
}

static int run_steps(const StepSet* ss, const void* x, void* y, cudaStream_t st) {
    for (auto& s : ss->steps) {
        int rc = s.run(st, x, y);
        if (rc != FD_OK) return fail(rc, std::string(fd_last_error()) + " [stage " + std::to_string(s.stage) + ": " + s.name + "]");
    }
    return FD_OK;
}

}  // namespace fd

// =========================================================================================
// C-ABI
// =========================================================================================
extern "C" {

int fd_abi_version(void) { return FD_ABI_VERSION; }
const char* fd_last_error(void) { return g_last_error.c_str(); }

int fd_plan_create(const fd_stage_desc* stages, int n_stages, int n, int h, int w, int dtype, int device, fd_plan** out) {
    if (!out) return fail(FD_ERR_INVALID, "out is NULL");
    *out = nullptr;
    if (!stages || n_stages < 3) return fail(FD_ERR_INVALID, "need at least stem + one block + head");
    if (n <= 0 || h <= 0 || w <= 0) return fail(FD_ERR_INVALID, "n, h, w must be positive");
    if (h % 32 || w % 32) return fail(FD_ERR_INVALID, "H and W must be multiples of 32 (skip shapes would not line up)");
    if (dtype != FD_F32 && dtype != FD_F16 && dtype != FD_BF16) return fail(FD_ERR_INVALID, "bad dtype");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0)
        return fail(FD_ERR_CUDA, "no CUDA device: fastdepth_b200 has no CPU fallback");
    if (device < 0 || device >= ndev) return fail(FD_ERR_INVALID, "bad device index");
    cudaDeviceProp prop{};
    FD_CUDA_OK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) return fail(FD_ERR_UNSUPPORTED, "fastdepth_b200 is built for sm_90a (H100) only");
    DeviceGuard guard(device);
    if (!guard.ok) return fail(FD_ERR_CUDA, "cudaSetDevice failed");

    std::vector<StageShape> shapes;
    int rc = walk_stages(stages, n_stages, n, h, w, shapes);
    if (rc != FD_OK) return rc;

    fd_plan* p = new fd_plan();
    p->n = n; p->h = h; p->w = w; p->dtype = dtype; p->device = device; p->n_sms = prop.multiProcessorCount;
    p->stages.resize(n_stages);
    const size_t es = dtype_size(dtype);
    for (int i = 0; i < n_stages; ++i) {
        Stage& s = p->stages[i];
        s.d = stages[i];
        const fd_stage_desc& d = s.d;
        s.g = shapes[i].g;
        s.out_h = shapes[i].out_h; s.out_w = shapes[i].out_w;
        s.out_c = shapes[i].out_c; s.out_pitch = s.out_c;
        if (d.kind != FD_STAGE_HEAD) {
            rc = dev_alloc(p, &s.out, (size_t)n * s.out_h * s.out_w * s.out_pitch * es);
            if (rc) break;
            s.out_alloc = s.out;
            if (d.skip_src >= 0 && d.skip_mode) {
                // concatenation (models.py:806-811): one wide NHWC buffer [.., c_out + c_skip]; this stage writes the channel
                // slice [0, c_out), the skip source is re-pointed to write (and be read by its consumer) in slice [c_out, ..).
                // The source's own dense buffer stays allocated (freed with the plan) but is no longer used
                Stage& src = p->stages[d.skip_src];
                src.out = static_cast<char*>(s.out) + (size_t)d.c_out * es;
                src.out_pitch = s.out_pitch;
                src.concat_src = i;
            }
        }
        if (d.kind == FD_STAGE_DWPW) {
            if ((rc = dev_alloc(p, &s.mid, (size_t)n * s.g.h_out * s.g.w_out * d.c_in * es))) break;
            if ((rc = dev_alloc(p, (void**)&s.dw_w, (size_t)d.ksize * d.ksize * d.c_in * 4))) break;
            if ((rc = dev_alloc(p, (void**)&s.dw_scale, (size_t)d.c_in * 4))) break;
            if ((rc = dev_alloc(p, (void**)&s.dw_bias, (size_t)d.c_in * 4))) break;
            if ((rc = dev_alloc(p, &s.pw_w, (size_t)d.c_in * d.c_out * es))) break;
        } else if (is_conv(d.kind)) {
            if ((rc = dev_alloc(p, &s.pw_w, (size_t)d.ksize * d.ksize * d.c_in * d.c_out * es))) break;
        } else if (d.kind == FD_STAGE_STEM) {
            if ((rc = dev_alloc(p, (void**)&s.pw_w_f32, (size_t)9 * d.c_in * d.c_out * 4))) break;
        } else {
            if ((rc = dev_alloc(p, (void**)&s.pw_w_f32, (size_t)d.c_in * 4))) break;
        }
        if ((rc = dev_alloc(p, (void**)&s.pw_scale, (size_t)d.c_out * 4))) break;
        if ((rc = dev_alloc(p, (void**)&s.pw_bias, (size_t)d.c_out * 4))) break;
    }
    if (rc != FD_OK) {
        std::string keep = g_last_error;
        fd_plan_destroy(p);
        g_last_error = keep;
        return rc;
    }
    *out = p;
    return FD_OK;
}

int fd_plan_set_stage_weights(fd_plan* p, int stage, const float* dw_w, const float* dw_scale, const float* dw_bias,
                              const float* pw_w, const float* pw_scale, const float* pw_bias) {
    if (!p) return fail(FD_ERR_INVALID, "plan is NULL");
    if (stage < 0 || stage >= (int)p->stages.size()) return fail(FD_ERR_INVALID, "bad stage index");
    if (!pw_w || !pw_scale || !pw_bias) return fail(FD_ERR_INVALID, "pw_w / pw_scale / pw_bias are required");
    DeviceGuard guard(p->device);
    Stage& s = p->stages[stage];
    const fd_stage_desc& d = s.d;
    if (d.kind == FD_STAGE_DWPW) {
        if (!dw_w || !dw_scale || !dw_bias) return fail(FD_ERR_INVALID, "block stage needs dw_w / dw_scale / dw_bias");
        const int kk = d.ksize * d.ksize;
        std::vector<float> t((size_t)kk * d.c_in);            // [c][k][k] -> [k*k][c]
        for (int c = 0; c < d.c_in; ++c)
            for (int j = 0; j < kk; ++j) t[(size_t)j * d.c_in + c] = dw_w[(size_t)c * kk + j];
        FD_CUDA_OK(cudaMemcpy(s.dw_w, t.data(), t.size() * 4, cudaMemcpyHostToDevice));
        FD_CUDA_OK(cudaMemcpy(s.dw_scale, dw_scale, (size_t)d.c_in * 4, cudaMemcpyHostToDevice));
        FD_CUDA_OK(cudaMemcpy(s.dw_bias, dw_bias, (size_t)d.c_in * 4, cudaMemcpyHostToDevice));
        int rc = upload_as_dtype(p->dtype, pw_w, (size_t)d.c_in * d.c_out, s.pw_w);
        if (rc) return rc;
    } else if (d.kind == FD_STAGE_CONV) {
        const int kk = d.ksize * d.ksize;
        std::vector<float> t((size_t)d.c_out * kk * d.c_in);   // [co][ci][ky][kx] -> [co][(ky,kx)][ci]
        for (int co = 0; co < d.c_out; ++co)
            for (int ci = 0; ci < d.c_in; ++ci)
                for (int j = 0; j < kk; ++j) t[((size_t)co * kk + j) * d.c_in + ci] = pw_w[((size_t)co * d.c_in + ci) * kk + j];
        int rc = upload_as_dtype(p->dtype, t.data(), t.size(), s.pw_w);
        if (rc) return rc;
    } else if (is_phased(d.kind)) {
        // DECONV [ci][co][ty][tx] / UPCONV [co][ci][ty][tx] -> [co][phase-major taps][ci]: phase q = 2 ry + rx holds its taps
        // sorted by (dy, dx), weight tap (convt_tap(ry, dy), convt_tap(rx, dx)) (fd_conv_plan.h)
        const int k = d.ksize, kk = k * k;
        ConvPhase ph[4];
        conv_phases(d.kind, k, ph);
        std::vector<float> t((size_t)d.c_out * kk * d.c_in);
        for (int q = 0; q < 4; ++q)
            for (int iy = 0; iy < ph[q].ny; ++iy)
                for (int ix = 0; ix < ph[q].nx; ++ix) {
                    const int tap = ph[q].tap0 + iy * ph[q].nx + ix;
                    const int wy = convt_tap(d.kind, k, q >> 1, ph[q].dy0 + iy), wx = convt_tap(d.kind, k, q & 1, ph[q].dx0 + ix);
                    for (int co = 0; co < d.c_out; ++co)
                        for (int ci = 0; ci < d.c_in; ++ci) {
                            const size_t src = d.kind == FD_STAGE_DECONV ? ((size_t)ci * d.c_out + co) * kk : ((size_t)co * d.c_in + ci) * kk;
                            t[((size_t)co * kk + tap) * d.c_in + ci] = pw_w[src + wy * k + wx];
                        }
                }
        int rc = upload_as_dtype(p->dtype, t.data(), t.size(), s.pw_w);
        if (rc) return rc;
    } else if (d.kind == FD_STAGE_STEM) {
        const int nk = 9 * d.c_in;
        std::vector<float> t((size_t)nk * d.c_out);            // [co][ci][ky][kx] -> [(ci,ky,kx)][co]
        for (int co = 0; co < d.c_out; ++co)
            for (int j = 0; j < nk; ++j) t[(size_t)j * d.c_out + co] = pw_w[(size_t)co * nk + j];
        FD_CUDA_OK(cudaMemcpy(s.pw_w_f32, t.data(), t.size() * 4, cudaMemcpyHostToDevice));
    } else {
        FD_CUDA_OK(cudaMemcpy(s.pw_w_f32, pw_w, (size_t)d.c_in * 4, cudaMemcpyHostToDevice));
        s.head_scale = pw_scale[0];
        s.head_bias = pw_bias[0];
    }
    FD_CUDA_OK(cudaMemcpy(s.pw_scale, pw_scale, (size_t)d.c_out * 4, cudaMemcpyHostToDevice));
    FD_CUDA_OK(cudaMemcpy(s.pw_bias, pw_bias, (size_t)d.c_out * 4, cudaMemcpyHostToDevice));
    s.have_weights = true;
    invalidate(p);
    return FD_OK;
}

static int* option_slot(fd_plan* p, const char* name) {
    if (!p || !name) return nullptr;
    if (!strcmp(name, "path")) return &p->opt_path;
    if (!strcmp(name, "fold_head")) return &p->opt_fold_head;
    if (!strcmp(name, "graph")) return &p->opt_graph;
    if (!strcmp(name, "tma_epilogue")) return &p->opt_tma_epilogue;
    if (!strcmp(name, "inplace_skip")) return &p->opt_inplace_skip;
    if (!strcmp(name, "pdl")) return &p->opt_pdl;
    if (!strcmp(name, "wait_sleep_ns")) return &p->opt_wait_sleep_ns;
    if (!strcmp(name, "chain")) return &p->opt_chain;
    if (!strcmp(name, "cluster")) return &p->opt_cluster;
    if (!strcmp(name, "tf32x3")) return &p->opt_tf32x3;
    if (!strcmp(name, "unfuse")) return &p->opt_unfuse;
    if (!strcmp(name, "front")) return &p->opt_front;
    return nullptr;
}

int fd_plan_set_option(fd_plan* p, const char* name, int value) {
    int* slot = option_slot(p, name);
    if (!slot) return fail(FD_ERR_INVALID, std::string("unknown option: ") + (name ? name : "(null)"));
    const bool is_time = !strcmp(name, "wait_sleep_ns");
    if (!strcmp(name, "unfuse")) {
        if (value < 0 || value > 2) return fail(FD_ERR_INVALID, "unfuse must be 0, 1 or 2");
    } else if (is_time ? (value < 0 || value > 100000) : (value != 0 && value != 1)) {
        return fail(FD_ERR_INVALID, is_time ? "wait_sleep_ns must be in [0, 100000]" : "option value must be 0 or 1");
    }
    if (*slot != value) { *slot = value; invalidate(p); }
    return FD_OK;
}

int fd_plan_get_option(fd_plan* p, const char* name, int* value) {
    int* slot = option_slot(p, name);
    if (!slot || !value) return fail(FD_ERR_INVALID, "unknown option or NULL value");
    *value = *slot;
    return FD_OK;
}

// The step set for (n, h, w), built on first use.  Beyond kMaxStepSets the least recently used set goes, with its graphs;
// the set of the plan's own (N, H, W) stays (introspection describes it).
static int ensure_steps(fd_plan* p, int n, int h, int w, StepSet** out) {
    StepSet* ss = find_set(p, n, h, w);
    if (!ss) {
        if (p->sets.size() >= kMaxStepSets) {
            size_t victim = p->sets.size();
            for (size_t i = 0; i < p->sets.size(); ++i)
                if (!is_capacity_set(p, p->sets[i]) && (victim == p->sets.size() || p->sets[i]->stamp < p->sets[victim]->stamp))
                    victim = i;
            const StepSet* v = p->sets[victim];
            for (size_t i = 0; i < p->graphs.size();)
                if (p->graphs[i].n == v->n && p->graphs[i].h == v->h && p->graphs[i].w == v->w) {
                    cudaGraphExecDestroy(p->graphs[i].exec);
                    p->graphs.erase(p->graphs.begin() + i);
                } else {
                    ++i;
                }
            destroy_set(p->sets[victim]);
            p->sets.erase(p->sets.begin() + victim);
        }
        ss = new StepSet();
        int rc = build_steps(p, n, h, w, ss);
        if (rc != FD_OK) { destroy_set(ss); return rc; }
        p->sets.push_back(ss);
    }
    ss->stamp = ++p->set_clock;
    *out = ss;
    return FD_OK;
}

static int forward_enqueue(fd_plan* p, const StepSet* ss, const void* x_dev, void* y_dev, cudaStream_t st);

int fd_forward(fd_plan* p, const void* x_dev, void* y_dev, void* stream) {
    if (!p) return fail(FD_ERR_INVALID, "NULL argument");
    return fd_forward_shape(p, p->n, p->h, p->w, x_dev, y_dev, stream);
}

int fd_forward_batch(fd_plan* p, int n, const void* x_dev, void* y_dev, void* stream) {
    if (!p) return fail(FD_ERR_INVALID, "NULL argument");
    return fd_forward_shape(p, n, p->h, p->w, x_dev, y_dev, stream);
}

int fd_forward_shape(fd_plan* p, int n, int h, int w, const void* x_dev, void* y_dev, void* stream) {
    if (!p) return fail(FD_ERR_INVALID, "NULL argument");
    if (h <= 0 || w <= 0 || h % 32 || w % 32)
        return fail(FD_ERR_INVALID, "h and w must be positive multiples of 32, got " + std::to_string(h) + "x" + std::to_string(w));
    // every stage buffer is dense NHWC of n * (h/s) * (w/s) * C elements, so any (n, h, w) with n*h*w <= N*H*W fits in its front
    const long long cap = (long long)p->n * p->h * p->w, per_image = (long long)h * w;
    const std::string plan_shape = std::to_string(p->n) + " x " + std::to_string(p->h) + " x " + std::to_string(p->w);
    if (per_image > cap)
        return fail(FD_ERR_INVALID, std::to_string(h) + "x" + std::to_string(w) + " needs " + std::to_string(per_image) +
                                        " pixels per image, more than the plan's capacity of " + std::to_string(cap) +
                                        " pixels (N x H x W = " + plan_shape + ")");
    if (n < 1 || n > cap / per_image)
        return fail(FD_ERR_INVALID, "batch size " + std::to_string(n) + " is outside [1, " + std::to_string(cap / per_image) +
                                        "] at " + std::to_string(h) + "x" + std::to_string(w) + ": the plan's capacity is " +
                                        std::to_string(cap) + " pixels (N x H x W = " + plan_shape + ")");
    if (!x_dev || !y_dev) return fail(FD_ERR_INVALID, "NULL argument");
    DeviceGuard guard(p->device);
    StepSet* ss = nullptr;
    int rc = ensure_steps(p, n, h, w, &ss);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    // A plan owns ONE set of activation buffers: a forward enqueued on another stream than the previous one first waits for that
    // one to finish (stream-ordered, no host synchronisation) instead of silently running into its intermediates.  Concurrency
    // is spelled with several plans (fastdepth_b200.engine.ForwardLanes).
    if (!p->last_done) FD_CUDA_OK(cudaEventCreateWithFlags(&p->last_done, cudaEventDisableTiming));
    if (p->last_stream_set && p->last_stream != st) FD_CUDA_OK(cudaStreamWaitEvent(st, p->last_done, 0));
    rc = forward_enqueue(p, ss, x_dev, y_dev, st);
    if (rc) return rc;
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(st, &cs) == cudaSuccess && cs == cudaStreamCaptureStatusNone) {
        FD_CUDA_OK(cudaEventRecord(p->last_done, st));
        p->last_stream = st; p->last_stream_set = true;
    }
    return FD_OK;
}

static int forward_enqueue(fd_plan* p, const StepSet* ss, const void* x_dev, void* y_dev, cudaStream_t st) {
    int rc = FD_OK;
    if (!p->opt_graph) return run_steps(ss, x_dev, y_dev, st);

    // Replay from a CUDA graph captured for this (x, y, n, h, w).
    for (auto& g : p->graphs)
        if (g.x == x_dev && g.y == y_dev && g.n == ss->n && g.h == ss->h && g.w == ss->w) {
            g.stamp = ++p->graph_clock;
            p->graph_misses = 0;
            FD_CUDA_OK(cudaGraphLaunch(g.exec, st));
            return FD_OK;
        }
    // A caller that never repeats an (x, y) pair (fresh output tensors that it keeps alive, a stream of distinct inputs) would
    // pay a capture + instantiate + eviction per call: after two cache-fulls of consecutive misses launch directly until a
    // pair repeats again (19 PDL-chained launches cost far less than one capture).
    if (++p->graph_misses > 2 * (int)kMaxGraphs) {
        if (p->graph_misses > (1 << 30)) p->graph_misses = 2 * (int)kMaxGraphs + 1;
        return run_steps(ss, x_dev, y_dev, st);
    }
    cudaStream_t cap;
    FD_CUDA_OK(cudaStreamCreateWithFlags(&cap, cudaStreamNonBlocking));
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    cudaError_t e = cudaStreamBeginCapture(cap, cudaStreamCaptureModeThreadLocal);
    if (e == cudaSuccess) {
        rc = run_steps(ss, x_dev, y_dev, cap);
        e = cudaStreamEndCapture(cap, &graph);
        if (rc == FD_OK && e == cudaSuccess) e = cudaGraphInstantiate(&exec, graph, 0);
    }
    if (graph) cudaGraphDestroy(graph);
    cudaStreamDestroy(cap);
    if (rc != FD_OK) return rc;
    if (e != cudaSuccess) return fail(FD_ERR_CUDA, std::string("graph capture: ") + cudaGetErrorString(e));
    if (p->graphs.size() >= kMaxGraphs) {
        size_t victim = 0;
        for (size_t i = 1; i < p->graphs.size(); ++i)
            if (p->graphs[i].stamp < p->graphs[victim].stamp) victim = i;
        cudaGraphExecDestroy(p->graphs[victim].exec);
        p->graphs.erase(p->graphs.begin() + victim);
    }
    p->graphs.push_back({x_dev, y_dev, ss->n, ss->h, ss->w, exec, ++p->graph_clock});
    FD_CUDA_OK(cudaGraphLaunch(exec, st));
    return FD_OK;
}

int fd_forward_host(fd_plan* p, const void* x_host, void* y_host, void* stream) {
    if (!p || !x_host || !y_host) return fail(FD_ERR_INVALID, "NULL argument");
    DeviceGuard guard(p->device);
    const size_t es = dtype_size(p->dtype);
    const size_t xb = (size_t)p->n * p->stages[0].d.c_in * p->h * p->w * es, yb = (size_t)p->n * p->h * p->w * es;
    if (!p->stage_x) {
        int rc = dev_alloc(p, &p->stage_x, xb);
        if (rc) return rc;
        if ((rc = dev_alloc(p, &p->stage_y, yb))) return rc;
    }
    cudaStream_t st = (cudaStream_t)stream;
    FD_CUDA_OK(cudaMemcpyAsync(p->stage_x, x_host, xb, cudaMemcpyHostToDevice, st));
    int rc = fd_forward(p, p->stage_x, p->stage_y, stream);
    if (rc) return rc;
    FD_CUDA_OK(cudaMemcpyAsync(y_host, p->stage_y, yb, cudaMemcpyDeviceToHost, st));
    FD_CUDA_OK(cudaStreamSynchronize(st));
    return FD_OK;
}

static const int kPipeSlots = 3;

int fd_pipeline_submit(fd_plan* p, const void* x_host, void* y_host, unsigned long long* ticket) {
    if (!p || !x_host || !y_host || !ticket) return fail(FD_ERR_INVALID, "NULL argument");
    DeviceGuard guard(p->device);
    const size_t es = dtype_size(p->dtype);
    const size_t xb = (size_t)p->n * p->stages[0].d.c_in * p->h * p->w * es, yb = (size_t)p->n * p->h * p->w * es;
    if (!p->pipe_h2d) {
        FD_CUDA_OK(cudaStreamCreateWithFlags(&p->pipe_h2d, cudaStreamNonBlocking));
        FD_CUDA_OK(cudaStreamCreateWithFlags(&p->pipe_run, cudaStreamNonBlocking));
        FD_CUDA_OK(cudaStreamCreateWithFlags(&p->pipe_d2h, cudaStreamNonBlocking));
        for (auto& sl : p->pipe) {
            int rc = dev_alloc(p, &sl.x, xb);
            if (rc) return rc;
            if ((rc = dev_alloc(p, &sl.y, yb))) return rc;
            FD_CUDA_OK(cudaEventCreateWithFlags(&sl.up, cudaEventDisableTiming));
            FD_CUDA_OK(cudaEventCreateWithFlags(&sl.done, cudaEventDisableTiming));
            FD_CUDA_OK(cudaEventCreateWithFlags(&sl.down, cudaEventDisableTiming));
        }
    }
    const unsigned long long t = p->pipe_next;
    fd_plan::PipeSlot& sl = p->pipe[t % kPipeSlots];
    if (sl.busy) {                                   // slot still owned by ticket t - kPipeSlots: wait for its download
        FD_CUDA_OK(cudaEventSynchronize(sl.down));
        sl.busy = false;
    }
    // upload on the copy-in stream; the forward waits for it; the download waits for the forward
    FD_CUDA_OK(cudaMemcpyAsync(sl.x, x_host, xb, cudaMemcpyHostToDevice, p->pipe_h2d));
    FD_CUDA_OK(cudaEventRecord(sl.up, p->pipe_h2d));
    FD_CUDA_OK(cudaStreamWaitEvent(p->pipe_run, sl.up, 0));
    int rc = fd_forward(p, sl.x, sl.y, p->pipe_run);
    if (rc) return rc;
    FD_CUDA_OK(cudaEventRecord(sl.done, p->pipe_run));
    FD_CUDA_OK(cudaStreamWaitEvent(p->pipe_d2h, sl.done, 0));
    FD_CUDA_OK(cudaMemcpyAsync(y_host, sl.y, yb, cudaMemcpyDeviceToHost, p->pipe_d2h));
    FD_CUDA_OK(cudaEventRecord(sl.down, p->pipe_d2h));
    // (a slot is only re-filled after the host saw its previous download complete, which implies its forward has
    //  finished reading sl.x -- no stream-level dependency is needed, and adding one would serialise the uploads)
    sl.busy = true;
    *ticket = t;
    p->pipe_next = t + 1;
    return FD_OK;
}

int fd_pipeline_wait(fd_plan* p, unsigned long long ticket) {
    if (!p) return fail(FD_ERR_INVALID, "NULL plan");
    if (ticket >= p->pipe_next) return fail(FD_ERR_INVALID, "unknown ticket");
    if (ticket + kPipeSlots < p->pipe_next) return FD_OK;        // its slot was already recycled, hence complete
    DeviceGuard guard(p->device);
    fd_plan::PipeSlot& sl = p->pipe[ticket % kPipeSlots];
    if (sl.busy) {
        FD_CUDA_OK(cudaEventSynchronize(sl.down));
        sl.busy = false;
    }
    return FD_OK;
}

int fd_stage_buffer(fd_plan* p, int stage, int which, void** dev_ptr, int* n, int* h, int* w, int* c, int* c_stride) {
    if (!p || stage < 0 || stage >= (int)p->stages.size() || !dev_ptr) return fail(FD_ERR_INVALID, "bad argument");
    Stage& s = p->stages[stage];
    const StepSet* full = find_set(p, p->n, p->h, p->w);
    int hh, ww, cc;
    void* ptr;
    if (which == 0) {
        ptr = full && full->runs[stage].out_eff ? full->runs[stage].out_eff : s.out; hh = s.out_h; ww = s.out_w; cc = s.g.c_out;
        // with decode_conv6 folded below the last upsample the last block writes its low-res output
        if (p->opt_fold_head && stage == (int)p->stages.size() - 2 && s.d.upsample && s.d.skip_src < 0) { hh = s.g.h_out; ww = s.g.w_out; }
    } else if (which == 1) {
        if (is_conv(s.d.kind)) return fail(FD_ERR_INVALID, "a CONV / DECONV / UPCONV stage has no depthwise intermediate");
        ptr = s.mid; hh = s.g.h_out; ww = s.g.w_out; cc = s.g.c_in;
    } else {
        return fail(FD_ERR_INVALID, "which must be 0 or 1");
    }
    if (!ptr) return fail(FD_ERR_STATE, "stage has no such buffer");
    *dev_ptr = ptr;
    if (n) *n = p->n;
    if (h) *h = hh;
    if (w) *w = ww;
    if (c) *c = cc;
    if (c_stride) *c_stride = (which == 0 && s.out_pitch > 0) ? s.out_pitch : cc;
    return FD_OK;
}

int fd_plan_launches_per_forward(fd_plan* p, int* n_launches) {
    if (!p || !n_launches) return fail(FD_ERR_INVALID, "NULL argument");
    DeviceGuard guard(p->device);
    StepSet* ss = nullptr;
    int rc = ensure_steps(p, p->n, p->h, p->w, &ss);
    if (rc) return rc;
    *n_launches = (int)ss->steps.size();
    return FD_OK;
}

int fd_plan_workspace_bytes(fd_plan* p, size_t* bytes) {
    if (!p || !bytes) return fail(FD_ERR_INVALID, "NULL argument");
    // the packed parameter copies of the plan's own step set are not counted; every other (n, h, w)'s set adds its own
    size_t sets = 0;
    for (const StepSet* ss : p->sets)
        if (!is_capacity_set(p, ss)) sets += ss->bytes;
    *bytes = p->workspace_bytes + p->split_bytes + sets;
    return FD_OK;
}

int fd_plan_step_count(fd_plan* p, int* n_steps) { return fd_plan_launches_per_forward(p, n_steps); }

int fd_plan_step_info(fd_plan* p, int step, int* stage, double* alg_bytes, double* macs, char* kernel_name, int name_cap) {
    if (!p) return fail(FD_ERR_INVALID, "NULL plan");
    DeviceGuard guard(p->device);
    StepSet* ss = nullptr;
    int rc = ensure_steps(p, p->n, p->h, p->w, &ss);
    if (rc) return rc;
    if (step < 0 || step >= (int)ss->steps.size()) return fail(FD_ERR_INVALID, "bad step index");
    const Step& s = ss->steps[step];
    if (stage) *stage = s.stage;
    if (alg_bytes) *alg_bytes = s.alg_bytes;
    if (macs) *macs = s.macs;
    if (kernel_name && name_cap > 0) {
        strncpy(kernel_name, s.name.c_str(), name_cap - 1);
        kernel_name[name_cap - 1] = 0;
    }
    return FD_OK;
}

int fd_plan_step_macs(fd_plan* p, int step, double* dw_macs, double* dense_macs) {
    if (!p) return fail(FD_ERR_INVALID, "NULL plan");
    DeviceGuard guard(p->device);
    StepSet* ss = nullptr;
    int rc = ensure_steps(p, p->n, p->h, p->w, &ss);
    if (rc) return rc;
    if (step < 0 || step >= (int)ss->steps.size()) return fail(FD_ERR_INVALID, "bad step index");
    const Step& s = ss->steps[step];
    if (dw_macs) *dw_macs = s.dw_macs;
    if (dense_macs) *dense_macs = s.macs - s.dw_macs;
    return FD_OK;
}

int fd_plan_time_steps(fd_plan* p, const void* x_dev, void* y_dev, void* stream, int warmup, int iters, int flush_l2,
                       float* ms_out) {
    if (!p || !x_dev || !y_dev || !ms_out || iters <= 0) return fail(FD_ERR_INVALID, "bad argument");
    DeviceGuard guard(p->device);
    StepSet* ss = nullptr;
    int rc = ensure_steps(p, p->n, p->h, p->w, &ss);
    if (rc) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (flush_l2 && !p->l2_flush) {
        p->l2_flush_bytes = size_t(256) << 20;               // > the 50 MB L2
        FD_CUDA_OK(cudaMalloc(&p->l2_flush, p->l2_flush_bytes));
    }
    rc = run_steps(ss, x_dev, y_dev, st);                     // make every intermediate valid
    if (rc) return rc;
    cudaEvent_t e0, e1;
    FD_CUDA_OK(cudaEventCreate(&e0));
    FD_CUDA_OK(cudaEventCreate(&e1));
    for (size_t i = 0; i < ss->steps.size() && rc == FD_OK; ++i) {
        for (int k = 0; k < warmup && rc == FD_OK; ++k) rc = ss->steps[i].run(st, x_dev, y_dev);
        float total = 0.f;
        for (int k = 0; k < iters && rc == FD_OK; ++k) {
            if (flush_l2) cudaMemsetAsync(p->l2_flush, k & 0xff, p->l2_flush_bytes, st);
            cudaEventRecord(e0, st);
            rc = ss->steps[i].run(st, x_dev, y_dev);
            cudaEventRecord(e1, st);
            cudaError_t e = cudaEventSynchronize(e1);
            if (e != cudaSuccess) { rc = fail(FD_ERR_CUDA, std::string("step ") + ss->steps[i].name + ": " + cudaGetErrorString(e)); break; }
            float ms = 0.f;
            cudaEventElapsedTime(&ms, e0, e1);
            total += ms;
        }
        ms_out[i] = total / iters;
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    return rc;
}

int fd_plan_trace_stage(fd_plan* p, int stage, void* y_dev, void* stream, unsigned long long* out_host, int cap, int* rows, int* cols) {
    if (!p || stage < 0 || stage >= (int)p->stages.size() || !out_host || !rows || !cols) return fail(FD_ERR_INVALID, "bad argument");
    DeviceGuard guard(p->device);
    StepSet* ss = nullptr;
    int rc = ensure_steps(p, p->n, p->h, p->w, &ss);
    if (rc) return rc;
    if (cap < 12 * 256) return fail(FD_ERR_INVALID, "trace buffer too small (need 3072 entries)");
    if (is_conv(p->stages[stage].d.kind)) return fail(FD_ERR_INVALID, "the stage timeline exists for fused block kernels only");
    const StageRun& r = ss->runs[stage];
    if (r.chain) return chain_tc_trace(r.chain, (cudaStream_t)stream, out_host, rows, cols);
    if (!r.tc) return fail(FD_ERR_STATE, "stage does not run the fused block kernel");
    return block_tc_trace(r.tc, (cudaStream_t)stream, y_dev, out_host, rows, cols);
}

int fd_debug_block_plan(int ksize, int stride, int h_out, int w_out, int n, int c_in, int c_out, int head, int* out, int cap) {
    if (!out || cap < 16) return fail(FD_ERR_INVALID, "need an int[16] output");
    const BlockPlanOut q = block_tc_debug_plan(ksize, stride, h_out, w_out, n, c_in, c_out, head);
    const int v[16] = {q.ok, q.splits, q.n_cta, q.items, q.kblocks, q.s_in, q.s_a, q.s_b, q.bn, q.nb, q.b_resident, q.n_stg,
                       q.smem_bytes, q.in_stage_stride, q.cs, q.dw_teams};
    for (int i = 0; i < 16; ++i) out[i] = v[i];
    return FD_OK;
}

int fd_debug_front_plan(const fd_stage_desc* stages, int n_stages, int dtype, int n, int h, int w, int* out, int cap) {
    if (!out || cap < 8) return fail(FD_ERR_INVALID, "need an int[8] output");
    if (!stages || n_stages < 1) return fail(FD_ERR_INVALID, "no stages");
    std::vector<StageShape> S;
    const int rc = walk_stages(stages, n_stages, n, h, w, S);
    if (rc != FD_OK) return rc;
    const bool ok = front_route_ok(stages, n_stages, dtype, S);
    out[0] = ok ? 1 : 0;
    out[1] = ok ? front_tc_items(n, h, w) : 0;
    front_tc_layout(S[0].g.c_in, out + 2);
    return FD_OK;
}

int fd_debug_conv_plan(int ksize, int h_out, int w_out, int n, int c_in, int c_out, int n_sms, int* out, int cap) {
    if (!out || cap < 16) return fail(FD_ERR_INVALID, "need an int[16] output");
    const ConvPlanOut q = conv_tc_debug_plan(FD_STAGE_CONV, ksize, h_out, w_out, n, c_in, c_out, n_sms);
    const int v[16] = {q.ok, q.ni, q.th, q.tw, q.bn, q.stages, q.m_tiles, q.n_splits, q.items, q.waves, q.kblocks, q.smem_bytes,
                       q.useful_permille, (int)(q.cost > 2e9 ? 2e9 : q.cost), 0, 0};
    for (int i = 0; i < 16; ++i) out[i] = v[i];
    return FD_OK;
}

int fd_debug_pw_plan(int h_out, int w_out, int n, int c_in, int c_out, int upsample, int n_sms, int* out, int cap) {
    if (!out || cap < 16) return fail(FD_ERR_INVALID, "need an int[16] output");
    const ConvPlanOut q = pw_tc_debug_plan(h_out, w_out, n, c_in, c_out, upsample, n_sms);
    const int v[16] = {q.ok, q.ni, q.th, q.tw, q.bn, q.stages, q.m_tiles, q.n_splits, q.items, q.waves, q.kblocks, q.smem_bytes,
                       q.useful_permille, (int)(q.cost > 2e9 ? 2e9 : q.cost), q.ok ? conv_stage_bytes(q.bn) : 0, 0};
    for (int i = 0; i < 16; ++i) out[i] = v[i];
    return FD_OK;
}

int fd_debug_pw_tf32x3_plan(int h_out, int w_out, int n, int c_in, int c_out, int upsample, int n_sms, int* out, int cap) {
    if (!out || cap < 16) return fail(FD_ERR_INVALID, "need an int[16] output");
    const ConvPlanOut q = pw_tf32x3_debug_plan(h_out, w_out, n, c_in, c_out, upsample, n_sms);
    const int v[16] = {q.ok, q.ni, q.th, q.tw, q.bn, q.stages, q.m_tiles, q.n_splits, q.items, q.waves, q.kblocks, q.smem_bytes,
                       q.useful_permille, (int)(q.cost > 2e9 ? 2e9 : q.cost), q.ok ? conv_stage_bytes_tf32x3(q.bn) : 0, 0};
    for (int i = 0; i < 16; ++i) out[i] = v[i];
    return FD_OK;
}

int fd_debug_conv_tf32x3_plan(int kind, int ksize, int h, int w, int n, int c_in, int c_out, int upsample, int n_sms, int* out,
                              int cap) {
    if (!out || cap < 44) return fail(FD_ERR_INVALID, "need an int[44] output");
    if (kind != FD_STAGE_CONV && !is_phased(kind)) return fail(FD_ERR_INVALID, "kind must be FD_STAGE_CONV, FD_STAGE_DECONV or FD_STAGE_UPCONV");
    const ConvPlanOut q = conv_tc_tf32x3_debug_plan(kind, ksize, h, w, n, c_in, c_out, upsample, n_sms);
    const int v[16] = {q.ok, q.ni, q.th, q.tw, q.bn, q.stages, q.m_tiles, q.n_splits, q.items, q.waves, q.kblocks, q.smem_bytes,
                       q.useful_permille, (int)(q.cost > 2e9 ? 2e9 : q.cost), q.ok ? conv_stage_bytes_tf32x3(q.bn) : 0, q.groups};
    for (int i = 0; i < 16; ++i) out[i] = v[i];
    for (int ph = 0; ph < 4; ++ph) {
        const int e[5] = {q.ph[ph].tap0, q.ph[ph].ny, q.ph[ph].nx, q.ph[ph].dy0, q.ph[ph].dx0};
        for (int j = 0; j < 5; ++j) out[16 + 5 * ph + j] = q.ok && ph < q.n_phases ? e[j] : 0;
    }
    for (int g = 0; g < 4; ++g)
        for (int j = 0; j < 2; ++j) out[36 + 2 * g + j] = q.ok ? q.group_ph[g][j] : -1;
    return FD_OK;
}

int fd_debug_convt_plan(int kind, int ksize, int h_in, int w_in, int n, int c_in, int c_out, int n_sms, int* out, int cap) {
    if (!out || cap < 44) return fail(FD_ERR_INVALID, "need an int[44] output");
    if (!is_phased(kind)) return fail(FD_ERR_INVALID, "kind must be FD_STAGE_DECONV or FD_STAGE_UPCONV");
    const ConvPlanOut q = conv_tc_debug_plan(kind, ksize, h_in, w_in, n, c_in, c_out, n_sms);
    const int v[16] = {q.ok, q.ni, q.th, q.tw, q.bn, q.stages, q.m_tiles, q.n_splits, q.items, q.waves, q.kblocks, q.smem_bytes,
                       q.useful_permille, (int)(q.cost > 2e9 ? 2e9 : q.cost), q.groups, 0};
    for (int i = 0; i < 16; ++i) out[i] = v[i];
    for (int ph = 0; ph < 4; ++ph) {
        const int e[5] = {q.ph[ph].tap0, q.ph[ph].ny, q.ph[ph].nx, q.ph[ph].dy0, q.ph[ph].dx0};
        for (int j = 0; j < 5; ++j) out[16 + 5 * ph + j] = q.ok ? e[j] : 0;
    }
    for (int g = 0; g < 4; ++g)
        for (int j = 0; j < 2; ++j) out[36 + 2 * g + j] = q.ok ? q.group_ph[g][j] : -1;
    return FD_OK;
}

int fd_metrics_accumulate(const void* pred_dev, const float* target_dev, int dtype, int n, int hw, double* sums_dev,
                          int device, void* stream) {
    if (!pred_dev || !target_dev || !sums_dev || n < 0 || hw <= 0) return fail(FD_ERR_INVALID, "bad argument");
    DeviceGuard guard(device);
    if (!guard.ok) return fail(FD_ERR_CUDA, "cudaSetDevice failed");
    return launch_metrics(dtype, pred_dev, target_dev, n, hw, sums_dev, (cudaStream_t)stream);
}

int fd_nyu_val_gather(const uint8_t* rgb_dev, const float* depth_dev, const int* rows_dev, const int* cols_dev, int n, int h_in,
                      int w_in, int out_h, int out_w, int dtype, void* x_dev, float* target_dev, int device, void* stream) {
    if (!rgb_dev || !rows_dev || !cols_dev || !x_dev || n < 0 || h_in <= 0 || w_in <= 0 || out_h <= 0 || out_w <= 0)
        return fail(FD_ERR_INVALID, "bad argument");
    if ((depth_dev == nullptr) != (target_dev == nullptr)) return fail(FD_ERR_INVALID, "depth and target must come together");
    DeviceGuard guard(device);
    if (!guard.ok) return fail(FD_ERR_CUDA, "cudaSetDevice failed");
    return launch_nyu_val_gather(dtype, rgb_dev, depth_dev, rows_dev, cols_dev, n, h_in, w_in, out_h, out_w, x_dev, target_dev,
                                 (cudaStream_t)stream);
}

void fd_plan_destroy(fd_plan* p) {
    if (!p) return;
    DeviceGuard guard(p->device);
    invalidate(p);
    for (auto& s : p->stages) {
        cudaFree(s.out_alloc ? s.out_alloc : s.out); cudaFree(s.mid); cudaFree(s.dw_w); cudaFree(s.dw_scale); cudaFree(s.dw_bias);
        cudaFree(s.pw_w); cudaFree(s.pw_w_f32); cudaFree(s.pw_scale); cudaFree(s.pw_bias);
    }
    for (auto& sl : p->pipe) {
        cudaFree(sl.x); cudaFree(sl.y);
        if (sl.up) cudaEventDestroy(sl.up);
        if (sl.done) cudaEventDestroy(sl.done);
        if (sl.down) cudaEventDestroy(sl.down);
    }
    if (p->last_done) cudaEventDestroy(p->last_done);
    if (p->pipe_h2d) cudaStreamDestroy(p->pipe_h2d);
    if (p->pipe_run) cudaStreamDestroy(p->pipe_run);
    if (p->pipe_d2h) cudaStreamDestroy(p->pipe_d2h);
    cudaFree(p->stage_x); cudaFree(p->stage_y); cudaFree(p->l2_flush);
    delete p;
}

}  // extern "C"
