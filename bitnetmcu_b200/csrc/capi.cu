// capi.cu -- the C ABI of include/bitnetmcu_b200.h: model container, batched inference (device + host
// pipelined), the four reference-named kernels and their batched forms.  No CPU compute path exists here:
// every entry needs a CUDA device and reports (or, for the reference-named symbols, aborts on) failure.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/bitnetmcu_b200.h"
#include "kernels.h"

using namespace bnm;

// -----------------------------------------------------------------------------------------------
// errors
// -----------------------------------------------------------------------------------------------
static thread_local std::string g_err;
static int fail(int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}
#define CU_TRY(expr)                                                                                       \
    do {                                                                                                   \
        cudaError_t e_ = (expr);                                                                           \
        if (e_ != cudaSuccess) return fail(-100 - (int)e_, "%s failed: %s", #expr, cudaGetErrorString(e_)); \
    } while (0)

enum { BNM_E_ARG = -1, BNM_E_NODEV = -2, BNM_E_UNSUPPORTED = -3, BNM_E_CUDA = -4 };

// the status of the kernels just launched: 0, or the launch error
static int launch_status() {
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail(BNM_E_CUDA, "kernel launch failed: %s", cudaGetErrorString(e));
}

static uint32_t round_up(uint32_t v, uint32_t m) { return (v + m - 1) / m * m; }

// For its scope, the calling thread may make the calls a stream capture in cudaStreamCaptureModeGlobal forbids to every other
// thread (allocation, stream synchronisation): the host paths' synchronous work runs under it, so that a host call next to
// another thread's capture neither fails nor invalidates that capture.  The thread's own mode comes back at the end of the scope
// (cudaThreadExchangeStreamCaptureMode, as PyTorch's allocator does).  None of that work touches a capturing stream.
struct RelaxedCaptureMode {
    cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
    RelaxedCaptureMode() { cudaThreadExchangeStreamCaptureMode(&mode); }
    ~RelaxedCaptureMode() { cudaThreadExchangeStreamCaptureMode(&mode); }
    RelaxedCaptureMode(const RelaxedCaptureMode &) = delete;
    RelaxedCaptureMode &operator=(const RelaxedCaptureMode &) = delete;
};

// the capture state of stream st (an eager stream when it cannot be read: a launch on it then reports the error)
static StreamCapture capture_of(cudaStream_t st) {
    StreamCapture c;
    cudaStreamCaptureStatus s = cudaStreamCaptureStatusNone;
    if (cudaStreamGetCaptureInfo(st, &s, &c.id) != cudaSuccess) {
        cudaGetLastError();
        return StreamCapture{};
    }
    c.active = s != cudaStreamCaptureStatusNone;   // an invalidated capture too: its launches must not enter the eager record
    return c;
}

// One allocation of T and its only owner, which frees it: device memory, or mapped pinned host memory (kPinned).  grow(need) makes
// it at least `need` bytes large: a larger request discards the contents and allocates anew (zeroed on request); one it already
// meets makes no CUDA call.
template <class T, bool kPinned>
struct Buffer {
    T *p = nullptr;
    size_t bytes = 0;
    Buffer() = default;
    Buffer(const Buffer &) = delete;
    Buffer &operator=(const Buffer &) = delete;
    ~Buffer() { release(); }
    void release() {
        if (p) kPinned ? cudaFreeHost(p) : cudaFree(p);
        p = nullptr;
        bytes = 0;
    }
    cudaError_t grow(size_t need, bool zero = false) {
        if (need <= bytes) return cudaSuccess;
        release();
        void *q = nullptr;
        cudaError_t e = kPinned ? cudaHostAlloc(&q, need, cudaHostAllocMapped) : cudaMalloc(&q, need);
        if (e != cudaSuccess) return e;
        p = static_cast<T *>(q);
        if (zero && (e = cudaMemset(p, 0, need)) != cudaSuccess) { release(); return e; }
        bytes = need;
        return cudaSuccess;
    }
};
template <class T> using DevBuf = Buffer<T, false>;
template <class T> using PinnedBuf = Buffer<T, true>;

// -----------------------------------------------------------------------------------------------
// model
// -----------------------------------------------------------------------------------------------
struct FcLayerHost {
    int32_t enc;
    uint32_t n_in, n_out;
    void *d_packed;
    size_t packed_bytes;
};

// one stream of the host pipeline (infer_pipelined) and its chunk's device copies, in bytes: images, logits or top-k scores,
// labels, top-k classes
struct PipeSlot {
    cudaStream_t stream = nullptr;
    DevBuf<char> d_images, d_logits, d_labels, d_classes;
};

// One staging generation of the small-batch path (infer_small): the rows of every call that joined it, in arrival order.
struct SmallGen {
    PinnedBuf<int8_t> h_in;     // [kSmallBatch][img_bytes]
    PinnedBuf<int32_t> h_out;   // logits [rows][n_classes] when a member asks for them, then labels [rows]: the kernels write
                                // them straight into this mapped memory
    DevBuf<int8_t> d_in;        // the device copy of h_in
    enum State { kOpen, kLaunched, kDone };
    // written under the batcher's lock; atomic so that a waiting caller may poll them without it (small_wait)
    std::atomic<int> state{kOpen};
    std::atomic<size_t> rows{0};   // rows reserved so far
    std::atomic<int> calls{0}, copied_in{0};
    int copied_out = 0;
    bool logits = false, labels = false;   // what the launch writes: what any member asks for
    int rc = 0;                 // the launch's result, and its error text, for every member
    std::string err;
};

// The small-batch path's shared state: calls that arrive while one generation's launch is in flight join the other, and the
// first of them launches it for all once that launch has completed.  All fields under mu.
struct SmallBatcher {
    std::mutex mu;
    std::condition_variable cv;
    SmallGen gen[2];
    std::atomic<int> open{0};             // the generation callers join
    std::atomic<bool> in_flight{false};   // a generation is launched and not yet complete
    cudaStream_t stream = nullptr;
};

struct bnm_model {
    int device = 0, sm_count = 0;
    int model_class = 0;
    uint32_t img_bytes = 256, n_classes = 0;
    std::vector<FcLayerHost> fc_host;
    std::vector<FcLayerDev> fc;
    // CNN front-end
    uint32_t channels = 0, xy0 = 0, feat_stride = 0;
    DevBuf<int8_t> d_conv[3];
    // options
    int opt_path = BNM_PATH_AUTO;
    int nf4_ext = 0;
    size_t chunk_images = 1 << 16;   // host pipeline chunk
    int launch_overlap = 0;
    int cnn_frontend = 0;            // BNM_OPT_CNN_FRONTEND
    long long conv3_bound = 0;       // static range of conv3's inputs for this model's weights (cnn_conv3_bound)
    bool conv3_fits_u16 = false;     // conv3_bound <= 65535: the tensor-core front-end runs conv3 on IDP.2A
    std::vector<int8_t> h_conv[3];   // host copies of the conv weights (range analysis)
    DevBuf<int> d_err;               // error word of the bounded device-side waits
    // fused plan
    FcChainPlan *plan = nullptr;
    std::string plan_err;
    uint32_t max_kpad = 0, max_nout = 0;   // the layer-by-layer path's scratch per image (LayerScratch)
    // the decoded FC planes and every call's device scratch come from this pool, stream-ordered (Scratch: on the call's stream)
    cudaMemPool_t pool = nullptr;
    // host pipeline: the large host calls take turns on host_mu
    std::mutex host_mu;
    PipeSlot slots[3];
    // small-batch path of bnm_infer_batch (the reference's own calling pattern: one image per Inference() call,
    // test_inference.py:146-150): pinned staging buffers, one stream, one synchronisation per shared launch
    SmallBatcher small;
    bool verbose = false;           // BNM_VERBOSE at model creation: the top-k entries name their route on every call
};
static const size_t kSmallBatch = 1024;

// bytes of an FC layer's packed weights, what the reference reads: n_out * ceil(n_in / weights per word) 32-bit words (ternary:
// n_out * (n_in / 10) uint16) -- inference.c:88-208.  An unknown encoding reads nothing and decodes as zeros (inference.c:202).
static size_t packed_weight_bytes(int32_t enc, uint32_t n_in, uint32_t n_out) {
    switch (enc) {
    case BNM_ENC_BINARY: return (size_t)n_out * ((n_in + 31) / 32) * 4;
    case BNM_ENC_2BITSYM: return (size_t)n_out * ((n_in + 15) / 16) * 4;
    case BNM_ENC_4BITSYM: case BNM_ENC_4BIT: case BNM_ENC_FP130: case BNM_ENC_NF4: return (size_t)n_out * ((n_in + 7) / 8) * 4;
    case BNM_ENC_8BIT: return (size_t)n_out * ((n_in + 3) / 4) * 4;
    case BNM_ENC_TERNARY: return (size_t)n_out * (n_in / 10) * 2;
    default: return 0;
    }
}

// an FC layer's decoded planes handed back to their pool on st, once the work enqueued on st before has used them
static void free_fc_layer(FcLayerDev &L, cudaStream_t st) {
    for (void *p : {(void *)L.dense_a, (void *)L.dense_b, (void *)L.quad_a, (void *)L.quad_b})
        if (p) cudaFreeAsync(p, st);
    L.dense_a = L.dense_b = nullptr;
    L.quad_a = L.quad_b = nullptr;
}

// one FC layer's packed weights (device, zero padded past the end) decoded into its int8 planes, the residual ones only where they
// are needed: stream-ordered allocations from `pool`, decoded on st and synchronised with it.  On failure nothing stays allocated.
static cudaError_t decode_fc_layer(const void *d_packed, int32_t enc, uint32_t n_in, uint32_t n_out, int nf4_ext, FcLayerDev &L,
                                   cudaMemPool_t pool, cudaStream_t st) {
    L.enc = enc;
    L.n_in = n_in;
    L.n_out = n_out;
    L.k_pad = round_up(std::max(n_in, 1u), 32);
    L.n_pad = round_up(n_out, 16);
    const size_t plane = (size_t)L.k_pad * L.n_pad;
    int *d_flag = nullptr;
    int flag = 0;
    cudaError_t e = cudaMallocFromPoolAsync(&L.dense_a, plane, pool, st);
    if (e == cudaSuccess) e = cudaMallocFromPoolAsync(&L.dense_b, plane, pool, st);
    if (e == cudaSuccess) e = cudaMallocFromPoolAsync(&L.quad_a, plane, pool, st);
    if (e == cudaSuccess) e = cudaMallocFromPoolAsync(&L.quad_b, plane, pool, st);
    if (e == cudaSuccess) e = cudaMallocFromPoolAsync(&d_flag, sizeof(int), pool, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(d_flag, 0, sizeof(int), st);
    if (e == cudaSuccess) {
        launch_decode_fc(d_packed, enc, n_in, n_out, L.k_pad, L.n_pad, L.dense_a, L.dense_b, L.quad_a, L.quad_b, nf4_ext, d_flag, st);
        e = cudaMemcpyAsync(&flag, d_flag, sizeof(int), cudaMemcpyDeviceToHost, st);
    }
    if (d_flag) cudaFreeAsync(d_flag, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) {
        free_fc_layer(L, st);
    } else if (!flag) {   // no residual plane needed (everything but FP130 layers that contain +128)
        cudaFreeAsync(L.dense_b, st);
        cudaFreeAsync(L.quad_b, st);
        L.dense_b = nullptr;
        L.quad_b = nullptr;
    }
    return e;
}

// the model's decoded layers (on the legacy stream: every caller has synchronised the device) and fused plan
static void free_fc_dev(bnm_model *m) {
    for (auto &L : m->fc) free_fc_layer(L, 0);
    m->fc.clear();
    if (m->plan) fc_chain_plan_destroy(m->plan);
    m->plan = nullptr;
}

static int effective_overlap(const bnm_model *m) {
    // the CNN front-end writes the features the FC kernel reads: there the dependency is real, never declare it away
    return m->model_class == BNM_MODEL_CNNMNIST && m->launch_overlap == 2 ? 1 : m->launch_overlap;
}

// decode all FC layers into int8 planes and (re)build the fused plan
static int build_fc_dev(bnm_model *m) {
    free_fc_dev(m);
    m->max_kpad = round_up(std::max(m->img_bytes, m->feat_stride), 32);
    m->max_nout = 0;
    for (auto &H : m->fc_host) {
        FcLayerDev L;
        if (cudaError_t e = decode_fc_layer(H.d_packed, H.enc, H.n_in, H.n_out, m->nf4_ext, L, m->pool, 0)) {   // nothing half-built stays behind
            free_fc_dev(m);
            return fail(BNM_E_CUDA, "weight decode of an FC layer failed: %s", cudaGetErrorString(e));
        }
        m->max_kpad = std::max(m->max_kpad, L.k_pad);
        m->max_nout = std::max(m->max_nout, L.n_out);
        m->fc.push_back(L);
    }
    m->n_classes = m->fc.back().n_out;
    // fused plan (may legitimately be unavailable for exotic shapes: the layered path then serves the model)
    char err[256] = {0};
    uint32_t in_bytes = m->model_class == BNM_MODEL_CNNMNIST ? m->feat_stride : m->img_bytes;
    m->plan = fc_chain_plan_create(m->fc.data(), (int)m->fc.size(), in_bytes, m->device, m->sm_count, m->verbose, err, sizeof(err));
    m->plan_err = err;
    fc_chain_plan_set_overlap(m->plan, effective_overlap(m));
    return 0;
}

// One call's device scratch: stream-ordered allocations from a pool (a model's, or the device's default one for the entries
// without a model) on the call's stream, handed back on that stream once the call has enqueued the work that uses them (the
// destructor).  Two calls in flight never share a byte of it, whatever their threads and streams, and no call waits on the host
// for another.  A model's pool keeps what it has (its release threshold is unbounded), so in steady state an allocation neither
// reaches the driver nor synchronises.
struct Scratch {
    cudaMemPool_t pool;
    cudaStream_t st;
    std::vector<void *> held;
    Scratch(cudaMemPool_t p, cudaStream_t s) : pool(p), st(s) {}
    Scratch(const Scratch &) = delete;
    Scratch &operator=(const Scratch &) = delete;
    ~Scratch() { for (void *p : held) cudaFreeAsync(p, st); }
    template <class T> cudaError_t get(T **p, size_t count) {   // count elements of T, null for none
        *p = nullptr;
        if (!count) return cudaSuccess;
        void *q = nullptr;
        cudaError_t e = cudaMallocFromPoolAsync(&q, count * sizeof(T), pool, st);
        if (e != cudaSuccess) return e;
        held.push_back(q);
        *p = static_cast<T *>(q);
        return cudaSuccess;
    }
};

// the layer-by-layer path's scratch for n images: int32 accumulators of the widest layer, ping-pong int8 activations
struct LayerScratch {
    int32_t *acc = nullptr;
    int8_t *act[2] = {nullptr, nullptr};
};
static cudaError_t layer_scratch(const bnm_model *m, Scratch &s, size_t n, LayerScratch &L) {
    cudaError_t e = s.get(&L.acc, n * std::max(m->max_nout, 1u));
    for (auto &a : L.act)
        if (e == cudaSuccess) e = s.get(&a, n * m->max_kpad);
    return e;
}

static int require_device_index(int device);

// -----------------------------------------------------------------------------------------------
// routes: the kernels a call runs on a model, and in what passes
// -----------------------------------------------------------------------------------------------
// Images per pass, each bounding the scratch of a call: 2^20 where a pass stages rows in scratch (scaled images, CNN features, the
// two-engine entry's labels), 2^17 for the C engine layer by layer, 65 536 (FC) / 2 048 (CNN: 2 x C kB of conv planes per image)
// for the emulator layer by layer.  A fused FC route that stages nothing runs one launch per pass of kFusedPass images: a launch
// takes at most 0x7fffff00 (its TMA row coordinate is an int32), and 2^28 costs one more launch per 64 GiB of 256-byte rows.
static const size_t kPass = 1 << 20, kLayerPass = 1 << 17, kEmulLayerPass[2] = {65536, 2048}, kFusedPass = 1 << 28;

enum Engine { kEngineC, kEngineEmul, kEngineBoth };
// the element type of a call's images: int8 (already scaled), float32, or 16-bit floats (section 11) of either format
enum InKind { kInI8, kInF32, kInF16, kInBF16 };
static_assert(kHalfFloat16 == BNM_FLOAT16 && kHalfBFloat16 == BNM_BFLOAT16, "HalfFormat follows the header's formats");
static size_t in_elem_bytes(InKind in) { return in == kInI8 ? 1 : in == kInF32 ? 4 : 2; }
static bool half_in(InKind in) { return in == kInF16 || in == kInBF16; }
static HalfFormat half_format(InKind in) { return in == kInBF16 ? kHalfBFloat16 : kHalfFloat16; }
// the stage that turns a pass of (scaled) images into the FC stage's int8 rows: none, the C engine's CNN front-end (the kernel
// cnn_frontend_kernel picks), the emulator's fused CNN front-end (k_cnn_emul_frontend on the float images, k_cnn_emul_frontend_i8
// on the scaled rows of a route that scales), or the layered emulator's expand / conv / renorm / pool / k_i32_to_i8
enum Front { kFrontNone, kFrontCnn, kFrontCnnEmul, kFrontCnnEmulLayers };

// A route: which kernels one call runs, chosen once per call (choose_route), named (print_route) and run (run_route) from this
// record alone.  Per pass of `pass` images, k_quantize_images (for its input kind) into scratch when `scale` (k_quantize_windows on the
// window scan's windows when `windows`: such a route always scales), then per `inner` images of
// that pass (0: all of it) the front-end, the FC stage and for a layered top-k k_topk_rows.  The FC stage is one launch of `form`,
// or the layer-by-layer chain with the engine's rule.  The two engines' route runs each engine's own route per pass instead.
struct Route {
    Engine engine;
    InKind in;
    bool topk;        // the k best classes out
    bool scale, windows;
    Front front;
    bool fused;
    FcForm form;
    size_t pass, inner;
};

// the route of an entry of `engine` on images of kind `in`, top-k or not, on this model with its options; windows: the float
// images are the windows of a stack of planes (the window scan: the engine's float route with k_quantize_windows as its scale
// step, never a fused float form; the emulator's fused CNN route then runs its front-end on the scaled rows).  16-bit images take
// the route of float32 ones, with the 16-bit float-input forms, or the 16-bit scaling kernel as the scale step.
static Route choose_route(const bnm_model *m, Engine engine, InKind in, bool topk, bool windows = false) {
    const bool fused = bnm_model_active_path(m) == BNM_PATH_TCGEN05, cnn = m->model_class == BNM_MODEL_CNNMNIST;
    const bool f32 = in != kInI8, half = half_in(in);
    Route r{engine, in, topk, false, windows, kFrontNone, fused, kFormInt8, 0, 0};
    // FC models whose plan has the engine's float-input form: one launch with the input scaling fused (no such top-k or window form)
    const FcForm float_form = engine == kEngineC ? (half ? kFormFloat16 : kFormFloat)
                              : engine == kEngineEmul ? (half ? kFormEmulFloat16 : kFormEmulFloat) : (half ? kFormEngines16 : kFormEngines);
    if (f32 && !topk && !windows && fused && !cnn && fc_chain_has_form(m->plan, float_form)) {
        r.form = float_form;
        r.pass = kFusedPass;
        return r;
    }
    if (engine == kEngineBoth) {
        r.fused = false;
        r.pass = kPass;
        return r;
    }
    if (engine == kEngineEmul) {   // float images only
        if (!fused || (cnn && m->channels > kCnnEmulMaxChannels)) {
            r.fused = false;
            r.scale = true;
            r.front = cnn ? kFrontCnnEmulLayers : kFrontNone;
            r.pass = kEmulLayerPass[cnn];
        } else {
            r.form = topk ? kFormEmulTopK : kFormEmulInt8;
            r.scale = !cnn || windows || half;   // 16-bit CNN images: k_cnn_emul_frontend_i8 on the scaled rows
            r.front = cnn ? kFrontCnnEmul : kFrontNone;
            r.pass = kPass;
        }
        return r;
    }
    r.form = topk ? kFormTopK : kFormInt8;
    r.front = cnn ? kFrontCnn : kFrontNone;
    r.pass = !fused ? kLayerPass : cnn ? kPass : kFusedPass;
    if (f32) {   // the int8 route on each pass of scaled images
        r.scale = true;
        r.inner = r.pass;
        r.pass = kPass;
    }
    return r;
}

// BNM_VERBOSE: "<what>: " and the kernels of route r.  The layered emulator names its chain only.
static void print_route(const bnm_model *m, const char *what, const Route &r) {
    if (!m->verbose) return;
    std::string s;
    const char *scale = r.in == kInF16 ? "k_quantize_images<float16> + " : r.in == kInBF16 ? "k_quantize_images<bfloat16> + " : "k_quantize_images + ";
    const char *windows = r.in == kInF16 ? "k_quantize_windows<float16> + " : r.in == kInBF16 ? "k_quantize_windows<bfloat16> + " : "k_quantize_windows + ";
    if (r.engine == kEngineBoth && !r.fused) {
        s = half_in(r.in) ? "bnm_infer_batch_device_f16 + bnm_emulate_batch_device_f16 + k_engine_counts"
                          : "bnm_infer_batch_device_f32 + bnm_emulate_batch_device + k_engine_counts";
    } else if (r.engine == kEngineEmul && !r.fused) {
        s = std::string(r.windows ? windows : "") + (r.topk ? "layer by layer + k_topk_rows<double>" : "layer by layer");
    } else {
        if (r.scale) s = r.windows ? windows : scale;
        if (r.front == kFrontCnn)
            s += cnn_frontend_kernel(m->channels, m->xy0, m->cnn_frontend) == kCnnFrontendTensorCores ? "k_cnn_frontend16_tc + " : "k_cnn_frontend16 + ";
        if (r.front == kFrontCnnEmul) s += r.scale ? "k_cnn_emul_frontend_i8 + " : "k_cnn_emul_frontend + ";
        s += r.fused ? fc_chain_form_name(m->plan, r.form) : r.topk ? "layer by layer + k_topk_rows<int32>" : "layer by layer";
    }
    fprintf(stderr, "bitnetmcu_b200: %s: %s\n", what, s.c_str());
}

extern "C" int bnm_version(void) { return BNM_VERSION; }
extern "C" const char *bnm_last_error(void) { return g_err.c_str(); }
extern "C" int bnm_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

extern "C" int bnm_model_create(int model_class, const bnm_layer *layers, uint32_t n_layers, uint32_t img_bytes, int device,
                                bnm_model **out) {
    if (!out || !layers || n_layers == 0) return fail(BNM_E_ARG, "bnm_model_create: null argument");
    *out = nullptr;
    if (model_class != BNM_MODEL_FCMNIST && model_class != BNM_MODEL_CNNMNIST)
        return fail(BNM_E_ARG, "unknown model class %d (expected MODEL_FCMNIST=0 / MODEL_CNNMNIST=1)", model_class);
    int ndev = bnm_device_count();
    if (ndev == 0) return fail(BNM_E_NODEV, "no CUDA device: this engine has no CPU fallback");
    if (device < 0 || device >= ndev) return fail(BNM_E_ARG, "device %d out of range (have %d)", device, ndev);
    CU_TRY(cudaSetDevice(device));
    cudaDeviceProp prop;
    CU_TRY(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9) return fail(BNM_E_UNSUPPORTED, "device %s is sm_%d%d; this library is built for sm_90a (Hopper) only", prop.name, prop.major, prop.minor);

    bnm_model *m = new bnm_model();
    m->device = device;
    m->sm_count = prop.multiProcessorCount;
    m->model_class = model_class;
    m->img_bytes = img_bytes ? img_bytes : 256;
    int rc = 0;
    uint32_t n_conv = 0;
    std::vector<uint32_t> front;   // kinds of the non-FC layers, in order
    for (uint32_t i = 0; i < n_layers && rc == 0; i++) {
        const bnm_layer &L = layers[i];
        if (L.kind == BNM_LAYER_FC) {
            if (!L.weights || L.n_in == 0 || L.n_out == 0) { rc = fail(BNM_E_ARG, "FC layer %u: empty", i); break; }
            const size_t need = packed_weight_bytes(L.bitperweight, L.n_in, L.n_out);
            if (L.weight_bytes < need) { rc = fail(BNM_E_ARG, "FC layer %u: %zu weight bytes, reference reads %zu", i, L.weight_bytes, need); break; }
            FcLayerHost H{L.bitperweight, L.n_in, L.n_out, nullptr, std::max<size_t>(need, 16)};
            if (cudaMalloc(&H.d_packed, H.packed_bytes + 16) != cudaSuccess) { rc = fail(BNM_E_CUDA, "cudaMalloc failed"); break; }
            cudaMemset(H.d_packed, 0, H.packed_bytes + 16);
            if (need) cudaMemcpy(H.d_packed, L.weights, need, cudaMemcpyHostToDevice);
            m->fc_host.push_back(H);
        } else if (L.kind == BNM_LAYER_CONV33) {
            front.push_back(L.kind);
            if (n_conv == 3) { rc = fail(BNM_E_UNSUPPORTED, "more than three conv layers"); break; }
            if (!L.weights || L.weight_bytes < (size_t)L.n_out * 9) { rc = fail(BNM_E_ARG, "conv layer %u: needs %u int8 weights", i, L.n_out * 9); break; }
            if (n_conv == 0) { m->channels = L.n_out; m->xy0 = L.n_in; }
            else if (L.n_out != m->channels) { rc = fail(BNM_E_UNSUPPORTED, "conv layers must share the channel count (dll.c:66)"); break; }
            if (m->d_conv[n_conv].grow((size_t)L.n_out * 9) != cudaSuccess) { rc = fail(BNM_E_CUDA, "cudaMalloc failed"); break; }
            cudaMemcpy(m->d_conv[n_conv].p, L.weights, (size_t)L.n_out * 9, cudaMemcpyHostToDevice);
            m->h_conv[n_conv].assign(static_cast<const int8_t *>(L.weights), static_cast<const int8_t *>(L.weights) + (size_t)L.n_out * 9);
            n_conv++;
        } else if (L.kind == BNM_LAYER_MAXPOOL22) {
            front.push_back(L.kind);
        } else {
            rc = fail(BNM_E_ARG, "layer %u: unknown kind %u", i, L.kind);
        }
    }
    if (rc == 0 && (m->fc_host.empty() || m->fc_host.size() > (size_t)kMaxFcLayers)) rc = fail(BNM_E_UNSUPPORTED, "model needs 1..%d FC layers", kMaxFcLayers);
    if (rc == 0 && model_class == BNM_MODEL_CNNMNIST) {
        const uint32_t want[5] = {BNM_LAYER_CONV33, BNM_LAYER_CONV33, BNM_LAYER_MAXPOOL22, BNM_LAYER_CONV33, BNM_LAYER_MAXPOOL22};
        if (front.size() != 5 || memcmp(front.data(), want, sizeof(want)) != 0)
            rc = fail(BNM_E_UNSUPPORTED, "CNN front-end must be conv,conv,pool,conv,pool (BitNetMCU_MNIST_dll.c:64-80)");
        else if (m->xy0 != 16 || m->img_bytes != 256)
            rc = fail(BNM_E_UNSUPPORTED, "CNN input must be 16x16 int8 (the reference hard-codes it, BitNetMCU_MNIST_dll.c:68)");
        else {
            uint32_t f = ((m->xy0 - 4) / 2 - 2) / 2;   // 16 -> 2
            m->feat_stride = round_up(m->channels * f * f, 16);
            m->conv3_bound = cnn_conv3_bound(m->h_conv[0].data(), m->h_conv[1].data(), m->channels);
            m->conv3_fits_u16 = m->conv3_bound <= 65535;
        }
    }
    if (rc == 0 && model_class == BNM_MODEL_FCMNIST && !front.empty()) rc = fail(BNM_E_ARG, "MODEL_FCMNIST with conv/pool layers");
    if (rc == 0) {
        cudaMemPoolProps props = {};
        props.allocType = cudaMemAllocationTypePinned;
        props.location.type = cudaMemLocationTypeDevice;
        props.location.id = device;
        uint64_t keep = UINT64_MAX;   // never hand memory back to the device: steady-state calls neither allocate nor synchronise
        if (cudaMemPoolCreate(&m->pool, &props) != cudaSuccess || cudaMemPoolSetAttribute(m->pool, cudaMemPoolAttrReleaseThreshold, &keep) != cudaSuccess)
            rc = fail(BNM_E_CUDA, "scratch memory pool: %s", cudaGetErrorString(cudaGetLastError()));
    }
    // before the plan: a rebuild (BNM_OPT_NF4_EXTENSION) keeps the diagnostics of the model's creation, whatever the environment then
    m->verbose = getenv("BNM_VERBOSE") != nullptr;
    if (rc == 0) rc = build_fc_dev(m);
    if (rc == 0 && m->d_err.grow(sizeof(int), true) != cudaSuccess) rc = fail(BNM_E_CUDA, "cudaMalloc failed");
    if (rc == 0) {
        for (auto &s : m->slots)
            if (cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking) != cudaSuccess) { rc = fail(BNM_E_CUDA, "cudaStreamCreate failed"); break; }
        if (rc == 0 && cudaStreamCreateWithFlags(&m->small.stream, cudaStreamNonBlocking) != cudaSuccess) rc = fail(BNM_E_CUDA, "cudaStreamCreate failed");
    }
    if (rc != 0) { std::string keep = g_err; bnm_model_destroy(m); g_err = keep; return rc; }
    if (m->verbose) {   // diagnostics: the routes of bnm_emulate_batch_device and bnm_compare_engines_device on the default path
        print_route(m, "emulator route", choose_route(m, kEngineEmul, kInF32, false));
        print_route(m, "engines route", choose_route(m, kEngineBoth, kInF32, false));
        // and which conv3 the tensor-core CNN front-end runs
        if (m->model_class == BNM_MODEL_CNNMNIST)
            fprintf(stderr, "bitnetmcu_b200: cnn front-end: conv3 bound %lld, conv3 on %s\n", m->conv3_bound,
                    m->conv3_fits_u16 ? "IDP.2A" : "IMAD");
    }
    *out = m;
    return 0;
}

extern "C" int bnm_model_load_blob(const void *blob, size_t bytes, int device, bnm_model **out) {
    // layout written by bitnetmcu_b200.model.Model.to_blob(): "BNM1" | class | n_layers | img_bytes | table | data
    if (!blob || bytes < 16 || memcmp(blob, "BNM1", 4) != 0) return fail(BNM_E_ARG, "not a BNM1 model blob");
    const uint8_t *b = static_cast<const uint8_t *>(blob);
    uint32_t hdr[3];
    memcpy(hdr, b + 4, 12);
    const uint32_t cls = hdr[0], n_layers = hdr[1], img_bytes = hdr[2];
    if (n_layers == 0 || n_layers > 64 || 16 + (size_t)n_layers * 32 > bytes) return fail(BNM_E_ARG, "corrupt model blob (layer table)");
    std::vector<bnm_layer> layers(n_layers);
    for (uint32_t i = 0; i < n_layers; i++) {
        uint32_t e[8];
        memcpy(e, b + 16 + (size_t)i * 32, 32);
        if ((size_t)e[6] + e[7] > bytes) return fail(BNM_E_ARG, "corrupt model blob (layer %u data)", i);
        layers[i] = bnm_layer{e[0], (int32_t)e[1], e[2], e[3], e[4], e[5], e[7] ? b + e[6] : nullptr, e[7]};
    }
    return bnm_model_create((int)cls, layers.data(), n_layers, img_bytes, device, out);
}

extern "C" void bnm_model_destroy(bnm_model *m) {
    if (!m) return;
    cudaSetDevice(m->device);
    cudaDeviceSynchronize();
    free_fc_dev(m);
    for (auto &H : m->fc_host) cudaFree(H.d_packed);
    for (auto &s : m->slots)
        if (s.stream) cudaStreamDestroy(s.stream);
    if (m->small.stream) cudaStreamDestroy(m->small.stream);
    // every call's scratch went back to it before the synchronisation above; the driver releases the pool once the planes'
    // frees enqueued by free_fc_dev have run
    if (m->pool) cudaMemPoolDestroy(m->pool);
    delete m;   // and with it the buffers it owns as members
}

extern "C" uint32_t bnm_model_n_classes(const bnm_model *m) { return m ? m->n_classes : 0; }
extern "C" uint32_t bnm_model_img_bytes(const bnm_model *m) { return m ? m->img_bytes : 0; }

extern "C" int bnm_model_active_path(const bnm_model *m) {
    if (!m) return 0;
    if (m->opt_path == BNM_PATH_LAYERS) return BNM_PATH_LAYERS;
    return m->plan ? BNM_PATH_TCGEN05 : BNM_PATH_LAYERS;
}

extern "C" int bnm_model_set_option(bnm_model *m, int option, int64_t value) {
    if (!m) return fail(BNM_E_ARG, "null model");
    CU_TRY(cudaSetDevice(m->device));
    switch (option) {
    case BNM_OPT_PATH:
        if (value < BNM_PATH_AUTO || value > BNM_PATH_TCGEN05) return fail(BNM_E_ARG, "bad path %lld", (long long)value);
        if (value == BNM_PATH_TCGEN05 && !m->plan) return fail(BNM_E_UNSUPPORTED, "fused tensor-core path unavailable for this model: %s", m->plan_err.c_str());
        m->opt_path = (int)value;
        return 0;
    case BNM_OPT_NF4_EXTENSION:
        if ((value != 0) == (m->nf4_ext != 0)) return 0;
        m->nf4_ext = value != 0;
        CU_TRY(cudaDeviceSynchronize());
        return build_fc_dev(m);
    case BNM_OPT_CHUNK_IMAGES:
        if (value < 128) return fail(BNM_E_ARG, "chunk must be >= 128 images");
        m->chunk_images = (size_t)value;
        return 0;
    case BNM_OPT_CNN_FRONTEND:
        if (value < 0 || value > 2) return fail(BNM_E_ARG, "CNN front-end must be 0 (auto), 1 (CUDA cores) or 2 (tensor cores)");
        if (value == 2 && !(m->model_class == BNM_MODEL_CNNMNIST && cnn_frontend_tc_supported(m->channels, m->xy0)))
            return fail(BNM_E_UNSUPPORTED, "tensor-core CNN front-end needs a 16x16 CNN model with a multiple of 16 (<= 128) channels");
        m->cnn_frontend = (int)value;
        return 0;
    case BNM_OPT_LAUNCH_OVERLAP:
        if (value < 0 || value > 2) return fail(BNM_E_ARG, "launch overlap mode must be 0, 1 or 2");
        m->launch_overlap = (int)value;
        fc_chain_plan_set_overlap(m->plan, effective_overlap(m));
        return 0;
    default:
        return fail(BNM_E_ARG, "unknown option %d", option);
    }
}
extern "C" int64_t bnm_model_get_option(const bnm_model *m, int option) {
    if (!m) return -1;
    switch (option) {
    case BNM_OPT_PATH: return m->opt_path;
    case BNM_OPT_NF4_EXTENSION: return m->nf4_ext;
    case BNM_OPT_CHUNK_IMAGES: return (int64_t)m->chunk_images;
    case BNM_OPT_LAUNCH_OVERLAP: return m->launch_overlap;
    case BNM_OPT_CNN_FRONTEND: return m->cnn_frontend;
    default: return -1;
    }
}

// -----------------------------------------------------------------------------------------------
// batched inference, device pointers
// -----------------------------------------------------------------------------------------------
// The FC chain layer by layer on int8 rows [n][stride]: per layer the dp4a kernel, per hidden layer the engine's renormalisation
// into the ping-pong activations.  The C engine writes the last layer's accumulators to logits (without them to the scratch, n x
// max_nout) and, for labels, takes its ReLUNorm's argmax; the emulator ends with k_emul_logits (float64 logits, labels).
static int run_layers(bnm_model *m, bool emul, const int8_t *act, uint32_t stride, size_t n, void *logits, uint32_t *labels,
                      const LayerScratch &ls, cudaStream_t st) {
    const size_t nl = m->fc.size();
    int32_t *acc = ls.acc;
    for (size_t l = 0; l < nl; l++) {
        const FcLayerDev &L = m->fc[l];
        if (l + 1 == nl && logits && !emul) acc = static_cast<int32_t *>(logits);
        if (!launch_fc_dp4a(act, stride, L, acc, n, st))
            return fail(BNM_E_UNSUPPORTED, "FC layer %zu: %u inputs need more shared memory than an SM has (layer kernel stages 128 rows)", l, L.n_in);
        if (l + 1 == nl) break;
        int8_t *next = ls.act[l & 1];   // the layered CNN emulator's features sit in act[1], dead once layer 0 has run
        stride = m->fc[l + 1].k_pad;
        if (emul) launch_relunorm_emul(acc, L.n_out, level_shift_of(L.enc), next, stride, n, st);   // BitNetMCU.py:528-530
        else launch_relunorm(acc, L.n_out, next, stride, nullptr, n, st);
        act = next;
    }
    const FcLayerDev &last = m->fc[nl - 1];
    if (emul) launch_emul_logits(acc, last.n_out, level_shift_of(last.enc), static_cast<double *>(logits), labels, n, st);
    else if (labels) launch_relunorm(acc, last.n_out, nullptr, 0, labels, n, st);
    return 0;
}

// CNN front-end into feat (int8 [n][feat_stride])
static int run_cnn_front(bnm_model *m, const int8_t *images, size_t n, int8_t *feat, cudaStream_t st) {
    if (launch_cnn_frontend(images, m->d_conv[0].p, m->d_conv[1].p, m->d_conv[2].p, m->channels, m->xy0, feat, m->feat_stride, n,
                            m->sm_count, m->cnn_frontend, m->d_err.p, m->conv3_fits_u16, st))
        return 0;
    return fail(BNM_E_UNSUPPORTED, "CNN front-end: %u channels at %ux%u not supported by the selected kernel (the reference hard-codes 16x16, dll.c:68)",
                m->channels, m->xy0, m->xy0);
}

// what a call writes from image b on (logits and scores: float64 for the emulator, else int32); its result-exchange rows in g
static FcOutputs outputs_from(const FcOutputs &o, size_t b, uint32_t n_classes, bool emul, GatherDst &g) {
    auto at = [&](void *p, size_t per_image) -> void * { return p ? static_cast<char *>(p) + b * per_image * (emul ? 8 : 4) : nullptr; };
    if (o.gather) {
        g = *o.gather;
        g.row_offset += b;
    }
    return FcOutputs{at(o.logits, n_classes), o.labels ? o.labels + b : nullptr, o.gather ? &g : nullptr,
                     {o.topk.k, o.topk.classes ? o.topk.classes + b * o.topk.k : nullptr, at(o.topk.scores, o.topk.k)}, o.engines};
}

// Route r (not the two engines' one) on n images on st, whose capture state is cap, arguments checked -> out: logits (int32
// [n][n_classes], float64 for the emulator), labels and gather; or with topk.k > 0 the k best classes of every image and their
// scores.  A fused route without a scale step or front-end allocates nothing; every other one runs through scratch of this
// call's own, for one pass (in a capture: graph-owned allocations, freed inside the graph).  A window route's images are the n windows of grid `win`
// in window order; its scale step reads them from the planes.
static int run_route(bnm_model *m, const Route &r, const void *images, size_t n, const FcOutputs &out, cudaStream_t st,
                     const StreamCapture &cap, const WindowGrid *win = nullptr) {
    const size_t pass = std::min(n, r.pass), inner = r.inner ? std::min(pass, r.inner) : pass;
    const bool emul = r.engine == kEngineEmul;
    const uint32_t elems = m->img_bytes, C = m->channels, k = out.topk.k;
    const size_t in_bytes = elems * in_elem_bytes(r.in);   // per input image
    Scratch s(m->pool, st);
    int8_t *q, *feat;     // a pass's scaled images; an inner pass's CNN features for the fused FC stage
    LayerScratch ls;      // the layer-by-layer chain's accumulators and activations
    double *lg;           // the layered emulator's top-k: its float64 logits
    int32_t *planes[2];   // the layered CNN emulator's int32 conv planes [(image, channel)][xy*xy]
    CU_TRY(s.get(&q, r.scale ? pass * elems : 0));
    CU_TRY(s.get(&feat, r.front == kFrontCnn || r.front == kFrontCnnEmul ? inner * m->feat_stride : 0));
    if (!r.fused) CU_TRY(layer_scratch(m, s, inner, ls));
    CU_TRY(s.get(&lg, emul && !r.fused && k ? inner * m->n_classes : 0));
    for (auto &p : planes) CU_TRY(s.get(&p, r.front == kFrontCnnEmulLayers ? inner * C * 256 : 0));
    GatherDst g;
    for (size_t b = 0; b < n; b += pass) {
        const size_t nb = std::min(pass, n - b);
        const char *in = r.windows ? nullptr : static_cast<const char *>(images) + b * in_bytes;
        size_t row_bytes = in_bytes;
        if (r.windows) {   // windows b .. b + nb - 1 of the stack, scaled as below
            if (!launch_quantize_windows(*win, b, nb, q, st))
                return fail(BNM_E_CUDA, "k_quantize_windows: cannot opt in to its dynamic shared memory");
            in = reinterpret_cast<const char *>(q);
            row_bytes = elems;
        } else if (r.scale) {   // test_inference.py:140-141, BitNetMCU.py:435-436
            if (half_in(r.in)) launch_quantize_images(reinterpret_cast<const uint16_t *>(in), half_format(r.in), elems, q, nb, st);
            else launch_quantize_images(reinterpret_cast<const float *>(in), elems, q, nb, st);
            in = reinterpret_cast<const char *>(q);
            row_bytes = elems;
        }
        for (size_t c = 0; c < nb; c += inner) {
            const size_t nc = std::min(inner, nb - c);
            const void *rows = in + c * row_bytes;   // the FC stage's input
            uint32_t stride = elems;
            int rc = 0;
            if (r.front == kFrontCnn) {
                if ((rc = run_cnn_front(m, static_cast<const int8_t *>(rows), nc, feat, st))) return rc;
            } else if (r.front == kFrontCnnEmul) {
                const bool ok = r.scale ? launch_cnn_emul_frontend_i8(static_cast<const int8_t *>(rows), m->d_conv[0].p, m->d_conv[1].p, m->d_conv[2].p, C, feat, m->feat_stride, nc, st)
                                        : launch_cnn_emul_frontend(static_cast<const float *>(rows), m->d_conv[0].p, m->d_conv[1].p, m->d_conv[2].p, C, feat, m->feat_stride, nc, st);
                if (!ok) return fail(BNM_E_CUDA, "emulator CNN front-end: cannot opt in to its dynamic shared memory");
            } else if (r.front == kFrontCnnEmulLayers) {
                // conv (ReLU, no shift) -> per-image renormalisation, pools in between (BitNetMCU.py:459-526)
                int32_t *p0 = planes[0], *p1 = planes[1];
                launch_expand_image(static_cast<const int8_t *>(rows), p0, C, 256, nc, st);
                launch_conv33relu(p0, m->d_conv[0].p, C, 16, 0, p1, nc * C, st);
                launch_conv_renorm(p1, C * 196, nc, st);
                launch_conv33relu(p1, m->d_conv[1].p, C, 14, 0, p0, nc * C, st);
                launch_conv_renorm(p0, C * 144, nc, st);
                launch_maxpool22(p0, 12, p1, nc * C, st);
                launch_conv33relu(p1, m->d_conv[2].p, C, 6, 0, p0, nc * C, st);
                launch_conv_renorm(p0, C * 16, nc, st);
                launch_maxpool22(p0, 4, p1, nc * C, st);
                launch_i32_to_i8(p1, C * 4, ls.act[1], m->feat_stride, nc, st);   // flatten (C, 2, 2) -> features (BitNetMCU.py:443-445)
            }
            if (r.front != kFrontNone) {
                rows = r.front == kFrontCnnEmulLayers ? ls.act[1] : feat;
                stride = m->feat_stride;
            }
            const FcOutputs o = outputs_from(out, b + c, m->n_classes, emul, g);
            if (r.fused) {
                // fed: the FC stage reads what this call's own scaling kernel or CNN front-end just wrote into its scratch.  Every
                // pass after a call's first is treated alike and keeps its wait: it reads and writes the same caller buffers as
                // the pass before it, and the mode-2 promise covers the call before this one, not the producer of these images
                // that the first pass may have waited for
                const bool fed = r.windows || r.scale || r.front != kFrontNone || b + c > 0;
                if ((rc = fc_chain_launch(m->plan, r.form, rows, nc, o, st, cap, fed, half_in(r.in) && !r.scale ? half_format(r.in) : 0)))
                    return fail(BNM_E_CUDA, "fused launch of %s failed (%d): %s", fc_chain_form_name(m->plan, r.form), rc,
                                cudaGetErrorString(cudaGetLastError()));
                continue;
            }
            if ((rc = run_layers(m, emul, static_cast<const int8_t *>(rows), stride, nc, emul && k ? lg : o.logits, o.labels, ls, st))) return rc;
            if (emul && k) launch_topk_rows(lg, m->n_classes, k, o.topk.classes, static_cast<double *>(o.topk.scores), nc, st);
            else if (k) launch_topk_rows(ls.acc, m->n_classes, k, o.topk.classes, static_cast<int32_t *>(o.topk.scores), nc, st);   // last layer's accumulators
        }
    }
    return launch_status();
}

extern "C" int bnm_infer_launch_count(const bnm_model *m, size_t n) {
    if (!m || n == 0) return 0;
    const Route r = choose_route(m, kEngineC, kInI8, false);
    const int per = (r.front != kFrontNone) + (r.fused ? 1 : (int)(2 * m->fc.size()));   // front-end, fc + relunorm per layer
    return (int)((n + r.pass - 1) / r.pass * per);
}

// -----------------------------------------------------------------------------------------------
// peer memory plumbing for the fused result exchange: cudaMalloc'd buffers exported / opened through CUDA IPC
// -----------------------------------------------------------------------------------------------
extern "C" int bnm_device_alloc(int device, size_t bytes, void **out) {
    if (!out) return fail(BNM_E_ARG, "bnm_device_alloc: null argument");
    *out = nullptr;
    if (int rc = require_device_index(device)) return rc;
    RelaxedCaptureMode relaxed;
    CU_TRY(cudaSetDevice(device));
    CU_TRY(cudaMalloc(out, bytes ? bytes : 16));
    return 0;
}
extern "C" void bnm_device_free(void *p) {
    RelaxedCaptureMode relaxed;
    if (p) cudaFree(p);
}
extern "C" int bnm_ipc_export(const void *dev_ptr, void *handle64) {
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handles are 64 bytes");
    if (!dev_ptr || !handle64) return fail(BNM_E_ARG, "bnm_ipc_export: null argument");
    cudaIpcMemHandle_t h;
    CU_TRY(cudaIpcGetMemHandle(&h, const_cast<void *>(dev_ptr)));
    memcpy(handle64, &h, 64);
    return 0;
}
extern "C" int bnm_ipc_open(int device, const void *handle64, void **out) {
    if (!handle64 || !out) return fail(BNM_E_ARG, "bnm_ipc_open: null argument");
    *out = nullptr;
    if (int rc = require_device_index(device)) return rc;
    CU_TRY(cudaSetDevice(device));
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    CU_TRY(cudaIpcOpenMemHandle(out, h, cudaIpcMemLazyEnablePeerAccess));
    return 0;
}
extern "C" int bnm_ipc_close(void *p) {
    if (!p) return 0;
    CU_TRY(cudaIpcCloseMemHandle(p));
    return 0;
}
// same-process multi-GPU callers: let `device` read / write memory of `peer` directly
extern "C" int bnm_enable_peer_access(int device, int peer) {
    if (int rc = require_device_index(device)) return rc;
    if (int rc = require_device_index(peer)) return rc;
    if (device == peer) return 0;
    int can = 0;
    CU_TRY(cudaDeviceCanAccessPeer(&can, device, peer));
    if (!can) return fail(BNM_E_UNSUPPORTED, "device %d cannot access device %d (no P2P path)", device, peer);
    CU_TRY(cudaSetDevice(device));
    cudaError_t e = cudaDeviceEnablePeerAccess(peer, 0);
    if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); return 0; }
    CU_TRY(e);
    return 0;
}

// -----------------------------------------------------------------------------------------------
// batched inference, host pointers: chunks round-robin over three streams so H2D, kernels and D2H overlap
// -----------------------------------------------------------------------------------------------
// Both generations' staging buffers, allocated by the first small call (under the batcher's lock): all of them or none.
static int small_buffers(bnm_model *m) {
    SmallGen *g = m->small.gen;
    if (g[1].d_in.p) return 0;
    CU_TRY(cudaSetDevice(m->device));
    const size_t in_bytes = kSmallBatch * (size_t)m->img_bytes, out_bytes = kSmallBatch * ((size_t)m->n_classes + 1) * 4;
    cudaError_t e = cudaSuccess;
    for (int i = 0; i < 2 && e == cudaSuccess; i++) {
        e = g[i].h_in.grow(in_bytes);
        if (e == cudaSuccess) e = g[i].h_out.grow(out_bytes);
        if (e == cudaSuccess) e = g[i].d_in.grow(in_bytes);
    }
    if (e == cudaSuccess) return 0;
    for (int i = 0; i < 2; i++) { g[i].h_in.release(); g[i].h_out.release(); g[i].d_in.release(); }
    return fail(-100 - (int)e, "small-batch staging buffers: %s", cudaGetErrorString(e));
}

// One generation's rows through the GPU: one copy in, one launch that writes the results into the mapped h_out, one
// synchronisation.
static int small_launch(bnm_model *m, SmallGen &g) {
    CU_TRY(cudaSetDevice(m->device));
    cudaStream_t st = m->small.stream;
    const size_t n = g.rows;
    int32_t *d_out;
    CU_TRY(cudaMemcpyAsync(g.d_in.p, g.h_in.p, n * (size_t)m->img_bytes, cudaMemcpyHostToDevice, st));
    CU_TRY(cudaHostGetDevicePointer(reinterpret_cast<void **>(&d_out), g.h_out.p, 0));
    const size_t n_log = g.logits ? n * (size_t)m->n_classes : 0;   // labels-only batches: the labels start the staging buffer
    uint32_t *d_lab = reinterpret_cast<uint32_t *>(d_out + n_log);
    const FcOutputs out{g.logits ? d_out : nullptr, g.labels ? d_lab : nullptr};
    if (int rc = run_route(m, choose_route(m, kEngineC, kInI8, false), g.d_in.p, n, out, st, StreamCapture{})) return rc;
    CU_TRY(cudaStreamSynchronize(st));
    return 0;
}

// Wait under lk until ready() holds.  A launch takes tens of microseconds and waking a sleeping thread about as long, and a
// sleeping caller that wakes must take the lock after every other one woken with it: so first poll ready() with the lock
// released for up to kSmallSpin, yielding the core, and only then sleep on cv.  ready() reads atomics only.
static const auto kSmallSpin = std::chrono::microseconds(200);
template <class Ready> static void small_wait(std::unique_lock<std::mutex> &lk, std::condition_variable &cv, Ready ready) {
    if (ready()) return;
    lk.unlock();
    const auto until = std::chrono::steady_clock::now() + kSmallSpin;
    while (!ready() && std::chrono::steady_clock::now() < until) std::this_thread::yield();
    lk.lock();
    cv.wait(lk, ready);
}

// n <= kSmallBatch images.  A call reserves rows in the open generation, copies its images in, and waits; the generation's first
// caller (its leader) launches it for all of them as soon as the other generation's launch has completed, so calls that arrive
// while a launch is in flight share the next one.  Then every caller copies its own rows out.  A caller alone on the model makes
// one copy, one launch and one synchronisation, as a plain call would; there is no timer.  Only the leader calls CUDA: a caller
// that joins a generation must never wait on the runtime while the launch in flight is being synchronised.  Like every host path
// it runs on the model's own streams, which are never captured (StreamCapture{}), in relaxed capture mode.
static int infer_small(bnm_model *m, const int8_t *images, size_t n, int32_t *logits, uint32_t *labels) {
    RelaxedCaptureMode relaxed;
    SmallBatcher &B = m->small;
    std::unique_lock<std::mutex> lk(B.mu);
    if (int rc = small_buffers(m)) return rc;
    small_wait(lk, B.cv, [&] { const SmallGen &o = B.gen[B.open]; return o.state == SmallGen::kOpen && o.rows + n <= kSmallBatch; });
    SmallGen &g = B.gen[B.open];
    const size_t row0 = g.rows;
    g.rows += n;
    const bool leader = g.calls++ == 0;
    g.logits = g.logits || logits;
    g.labels = g.labels || labels;
    lk.unlock();
    memcpy(g.h_in.p + row0 * m->img_bytes, images, n * (size_t)m->img_bytes);
    lk.lock();
    g.copied_in++;
    B.cv.notify_all();
    if (leader) {
        small_wait(lk, B.cv, [&] { return !B.in_flight; });   // the generation takes callers until the launch before it has completed
        g.state = SmallGen::kLaunched;
        B.open ^= 1;
        B.in_flight = true;
        small_wait(lk, B.cv, [&] { return g.copied_in == g.calls; });
        lk.unlock();
        const int rc = small_launch(m, g);
        lk.lock();
        g.rc = rc;
        g.err = rc ? g_err : std::string();
        g.state = SmallGen::kDone;
        B.in_flight = false;
        if (m->verbose && g.calls > 1) fprintf(stderr, "bitnetmcu_b200: small batch: %zu images from %d calls\n", g.rows.load(), g.calls.load());
        B.cv.notify_all();
    } else {
        small_wait(lk, B.cv, [&] { return g.state == SmallGen::kDone; });
    }
    const int rc = g.rc;
    if (rc) g_err = g.err;   // every member reports the launch's failure in its own thread
    const size_t n_log = g.logits ? g.rows * (size_t)m->n_classes : 0;
    lk.unlock();
    if (!rc && logits) memcpy(logits, g.h_out.p + row0 * m->n_classes, n * (size_t)m->n_classes * 4);
    if (!rc && labels) memcpy(labels, g.h_out.p + n_log + row0, n * 4);
    lk.lock();
    if (++g.copied_out == g.calls) {   // the last member out opens the generation again
        g.state = SmallGen::kOpen;
        g.rows = 0;
        g.calls = g.copied_in = g.copied_out = 0;
        g.logits = g.labels = false;
        B.cv.notify_all();
    }
    return rc;
}

// A band of a host window scan (section 14): window rows row .. row + rows - 1 of planes plane .. plane + planes - 1 (several
// planes: whole ones, rows == out_h), its windows contiguous in window order.
struct WindowBand {
    size_t plane, planes;
    uint32_t row, rows;
};
static const size_t kBandWindows = kPass;   // windows per band at most: the window route's pass

// the page rows [*a, *e) that window rows r0 .. r1 - 1 of page grid g read (the first window row of a plane starts at page row
// -top): the rows their windows cover and, with reflect, down to the mirror image of the topmost border row they read, which the
// windows need not cover (out_h * stride_y small next to top).  The bottom border's mirror rows are covered by the band rule
static void band_rows(const WindowGrid &g, uint32_t r0, uint32_t r1, long long *a, long long *e) {
    const long long y0 = (long long)r0 * g.stride_y - g.top;   // the first window's first page row
    *a = std::max(0ll, y0);
    *e = std::min((long long)g.height, (long long)(r1 - 1) * g.stride_y - g.top + 16);
    if (g.pad_mode == kPadReflect && y0 < 0) *e = std::max(*e, std::min((long long)g.height, 1 - y0));
}

// The bands of page grid g (of elem-byte pixels) at `budget` bytes of page pixels per band: the rule of the header's section 14.
// Each band's rows contain every page row its windows read, the border rows that replicate or reflect padding maps onto included.
static std::vector<WindowBand> window_bands(const WindowGrid &g, size_t elem, size_t budget) {
    std::vector<WindowBand> bands;
    const size_t row_bytes = (size_t)g.width * elem, plane_windows = (size_t)g.out_h * g.out_w;
    long long a, e;
    band_rows(g, 0, g.out_h, &a, &e);
    const size_t plane_bytes = (size_t)(e - a) * row_bytes;
    if (plane_bytes <= budget && plane_windows <= kBandWindows) {   // runs of whole planes
        const size_t per = std::min(budget / plane_bytes, kBandWindows / plane_windows);
        for (size_t p = 0; p < g.planes; p += per) bands.push_back({p, std::min(per, g.planes - p), 0, g.out_h});
        return bands;
    }
    const long long sy = g.stride_y, top = g.top, H = g.height;
    const long long by_bytes = ((long long)(budget / row_bytes) - 16) / sy + 1;   // may be < 1: one window row is the least
    const size_t R = (size_t)std::max(1ll, std::min(by_bytes, (long long)(kBandWindows / g.out_w)));
    // the first band: every window row that starts in the top border (band_rows adds the rows reflect mirrors them onto)
    const size_t head = (size_t)((top + sy - 1) / sy);
    // t: the band holding window row t runs to the plane's end (none when no window reaches below the page)
    size_t t = g.out_h;
    const long long over = (long long)(g.out_h - 1) * sy - top + 16 - H;   // rows the last window reaches below the page
    if (over > 0) {
        t = H + top >= 16 ? (size_t)((H + top - 16) / sy + 1) : 0;   // the first row reaching into the bottom border
        if (g.pad_mode == kPadReflect) t = std::min(t, (size_t)((H - 1 - over + top) / sy));
    }
    for (size_t p = 0; p < g.planes; p++)
        for (size_t s = 0, end; s < g.out_h; s = end) {
            end = s ? s + R : std::max(R, head);
            if (end > t || end >= g.out_h) end = g.out_h;
            bands.push_back({p, 1, (uint32_t)s, (uint32_t)(end - s)});
        }
    return bands;
}

// Route r (not the two engines' one) on host buffers, each unit through one slot's buffers: its input in, run_route, out's arrays
// back, those copies enqueued after the next unit's input and kernels so that a pageable destination, which blocks the thread
// until its copy is done, does not hold up the next unit.  The units are chunks of chunk_images images, or with win the bands of
// the window scan of the host pages of grid win (window_bands), each band's page rows copied into the slot's staging and scanned
// there through a grid shifted to the band.  Synchronous.  name: the entry, for the band line under BNM_VERBOSE.
static int infer_pipelined(bnm_model *m, const Route &r, const void *images, size_t n, const FcOutputs &out,
                           const WindowGrid *win = nullptr, const char *name = nullptr) {
    RelaxedCaptureMode relaxed;
    std::lock_guard<std::mutex> turn(m->host_mu);   // large host calls take turns: each one keeps the copy engines busy alone
    const size_t chunk = std::min(n, m->chunk_images), k = out.topk.k;
    // per image, in bytes: the images (float32 or int8), d_logits the logits or the top-k scores (float64 for the emulator, else
    // int32; bnm_infer_batch sizes it and d_labels whether or not it takes them), d_labels the label, d_classes the top-k classes
    const size_t in_bytes = in_elem_bytes(r.in) * m->img_bytes, el = r.engine == kEngineEmul ? 8 : 4;
    const size_t logit_bytes = (k ? (out.topk.scores ? k : 0) : m->n_classes) * el, label_bytes = k ? 0 : 4, class_bytes = k * 4;
    // a window scan's bands, and its staging rows: the page's, rounded up to 16 bytes
    const size_t px = in_elem_bytes(r.in), dpitch = win ? round_up(win->width, 16 / (uint32_t)px) : 0;
    std::vector<WindowBand> bands;
    size_t units = (n + chunk - 1) / chunk, items = chunk, staged = chunk * in_bytes;   // per unit at most: images or windows, bytes
    if (win) {
        bands = window_bands(*win, px, m->chunk_images * 1024);
        units = bands.size();
        items = staged = 0;
        for (const auto &b : bands) {
            long long a, e;
            band_rows(*win, b.row, b.row + b.rows, &a, &e);
            items = std::max(items, b.planes * b.rows * win->out_w);
            staged = std::max(staged, b.planes * (size_t)(e - a) * dpitch * px);
        }
        if (m->verbose) print_route(m, ("host windows: " + std::string(name) + ": " + std::to_string(units) + " bands").c_str(), r);
    }
    bool small = false;
    for (auto &s : m->slots)
        small = small || s.d_images.bytes < staged || s.d_classes.bytes < items * class_bytes ||
                s.d_logits.bytes < items * logit_bytes || s.d_labels.bytes < items * label_bytes;
    if (small) {
        for (auto &s : m->slots) CU_TRY(cudaStreamSynchronize(s.stream));   // no chunk of an earlier call may still use a buffer that is reallocated
        for (auto &s : m->slots) {
            CU_TRY(s.d_images.grow(staged));
            CU_TRY(s.d_classes.grow(items * class_bytes));
            CU_TRY(s.d_logits.grow(items * logit_bytes));
            CU_TRY(s.d_labels.grow(items * label_bytes));
        }
    }
    // every unit's scratch is its own (run_route): the units of every path overlap in time on all three streams
    char *h_logits = static_cast<char *>(k ? out.topk.scores : out.logits);   // where d_logits goes
    auto copy_out = [&](PipeSlot &s, size_t b, size_t nb) -> int {   // items b .. b + nb - 1 from slot s
        if (k) CU_TRY(cudaMemcpyAsync(out.topk.classes + b * k, s.d_classes.p, nb * class_bytes, cudaMemcpyDeviceToHost, s.stream));
        if (h_logits) CU_TRY(cudaMemcpyAsync(h_logits + b * logit_bytes, s.d_logits.p, nb * logit_bytes, cudaMemcpyDeviceToHost, s.stream));
        if (out.labels) CU_TRY(cudaMemcpyAsync(out.labels + b, s.d_labels.p, nb * 4, cudaMemcpyDeviceToHost, s.stream));
        return 0;
    };
    PipeSlot *prev = nullptr;
    size_t prev_b = 0, prev_nb = 0;
    for (size_t u = 0, b = 0; u < units; u++) {
        PipeSlot &s = m->slots[u % 3];
        size_t nb = std::min(chunk, n - b);
        WindowGrid band;   // the window scan: the band's rows in the slot's staging
        if (win) {
            const WindowBand &B = bands[u];
            long long a, e;
            band_rows(*win, B.row, B.row + B.rows, &a, &e);
            const size_t rows = (size_t)(e - a), spitch = win->pitch * px;
            const char *src = static_cast<const char *>(win->image) + (B.plane * win->plane_pitch + (size_t)a * win->pitch) * px;
            if (B.planes > 1 && rows == win->height && win->plane_pitch == win->height * win->pitch)   // one run of rows
                CU_TRY(cudaMemcpy2DAsync(s.d_images.p, dpitch * px, src, spitch, win->width * px, B.planes * rows, cudaMemcpyHostToDevice, s.stream));
            else
                for (size_t p = 0; p < B.planes; p++)
                    CU_TRY(cudaMemcpy2DAsync(s.d_images.p + p * rows * dpitch * px, dpitch * px, src + p * win->plane_pitch * px, spitch,
                                             win->width * px, rows, cudaMemcpyHostToDevice, s.stream));
            band = *win;
            band.image = s.d_images.p;
            band.planes = (uint32_t)B.planes;
            band.height = (uint32_t)rows;
            band.pitch = dpitch;
            band.plane_pitch = B.planes > 1 ? rows * dpitch : 0;
            band.out_h = B.rows;
            band.top = (uint32_t)(a - ((long long)B.row * win->stride_y - win->top));   // > 0 in a plane's first band only
            nb = B.planes * B.rows * win->out_w;
        } else {
            CU_TRY(cudaMemcpyAsync(s.d_images.p, static_cast<const char *>(images) + b * in_bytes, nb * in_bytes, cudaMemcpyHostToDevice, s.stream));
        }
        uint32_t *d_labels = reinterpret_cast<uint32_t *>(s.d_labels.p), *d_classes = reinterpret_cast<uint32_t *>(s.d_classes.p);
        const FcOutputs d{out.logits ? s.d_logits.p : nullptr, out.labels ? d_labels : nullptr, nullptr,
                         {(uint32_t)k, d_classes, out.topk.scores ? s.d_logits.p : nullptr}};
        if (int rc = run_route(m, r, s.d_images.p, nb, d, s.stream, StreamCapture{}, win ? &band : nullptr)) return rc;
        if (prev)
            if (int rc = copy_out(*prev, prev_b, prev_nb)) return rc;
        prev = &s;
        prev_b = b;
        prev_nb = nb;
        b += nb;
    }
    if (prev)
        if (int rc = copy_out(*prev, prev_b, prev_nb)) return rc;
    for (auto &s : m->slots) CU_TRY(cudaStreamSynchronize(s.stream));
    return 0;
}

extern "C" void *bnm_host_alloc(size_t bytes) {
    RelaxedCaptureMode relaxed;
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); fail(BNM_E_CUDA, "cudaHostAlloc(%zu) failed", bytes); return nullptr; }
    return p;
}
extern "C" void bnm_host_free(void *p) {
    RelaxedCaptureMode relaxed;
    if (p) cudaFreeHost(p);
}

// -----------------------------------------------------------------------------------------------
// the four kernels, batched over host buffers
// -----------------------------------------------------------------------------------------------
static int require_device() {
    if (bnm_device_count() == 0) return fail(BNM_E_NODEV, "no CUDA device: this engine has no CPU fallback");
    return 0;
}
static int require_device_index(int device) {
    const int n = bnm_device_count();
    if (n == 0) return fail(BNM_E_NODEV, "no CUDA device: this engine has no CPU fallback");
    if (device < 0 || device >= n) return fail(BNM_E_ARG, "device %d out of range (have %d)", device, n);
    return 0;
}

// The stream of the entries without a model (the four kernels' batched forms, bnm_quantize_images) on the current device: one
// non-blocking stream per device, created by the first such call and kept for the process.  Their copies and kernels run on it
// and they wait for it alone, so they neither wait for nor hold up the legacy stream or a capture on another stream.
static int host_stream(cudaStream_t *st) {
    static std::mutex mu;
    static std::vector<cudaStream_t> streams;
    int dev = 0;
    CU_TRY(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lock(mu);
    if ((size_t)dev >= streams.size()) streams.resize(dev + 1, nullptr);
    if (!streams[dev]) CU_TRY(cudaStreamCreateWithFlags(&streams[dev], cudaStreamNonBlocking));
    *st = streams[dev];
    return 0;
}

// The device side of a host call without a model: Scratch from the device's default memory pool on its host stream, each buffer
// copied from host memory (in) or, once the entry's kernels have run, to it (out).
struct HostStaging : Scratch {
    struct Copy { void *host; const void *dev; size_t bytes; };
    std::vector<Copy> outs;
    using Scratch::Scratch;
    template <class T> cudaError_t in(T **d, const T *h, size_t count) {   // count elements of h
        cudaError_t e = get(d, count);
        return e != cudaSuccess || !count ? e : cudaMemcpyAsync(*d, h, count * sizeof(T), cudaMemcpyHostToDevice, st);
    }
    template <class T> cudaError_t out(T **d, T *h, size_t count) {   // count elements for h; null h: a buffer nothing copies out
        cudaError_t e = get(d, count);
        if (e == cudaSuccess && h && count) outs.push_back({h, *d, count * sizeof(T)});
        return e;
    }
};

// A host call without a model, its arguments checked, on the current device in relaxed capture mode: body(s) stages its inputs
// in s and enqueues its kernels on s.st (the device's host stream); then the launch status, the copies out and one
// synchronisation of that stream.  Every temporary is stream-ordered, so the call waits for its own stream and never for the
// device.
template <class Body> static int host_call(Body body) {
    RelaxedCaptureMode relaxed;   // outlives the staging: its frees run under it
    int dev = 0;
    cudaStream_t st;
    cudaMemPool_t pool;
    CU_TRY(cudaGetDevice(&dev));
    CU_TRY(cudaDeviceGetDefaultMemPool(&pool, dev));
    if (int rc = host_stream(&st)) return rc;
    HostStaging s(pool, st);
    if (int rc = body(s)) return rc;
    CU_TRY(cudaGetLastError());
    for (const auto &c : s.outs) CU_TRY(cudaMemcpyAsync(c.host, c.dev, c.bytes, cudaMemcpyDeviceToHost, st));
    CU_TRY(cudaStreamSynchronize(st));
    return 0;
}

extern "C" int bnm_processfclayer_batch(const int8_t *activations, const uint32_t *weights, int32_t enc, uint32_t n_input,
                                        uint32_t n_output, int32_t *output, size_t n, int nf4_extension) {
    if (int rc = require_device()) return rc;
    if (n == 0 || n_output == 0) return 0;
    if (!activations || !weights || !output) return fail(BNM_E_ARG, "bnm_processfclayer_batch: null argument");
    // Ternary layers declare n_input padded to a multiple of 10 with zero trits (exportquant.py:132-137,166) and the
    // reference never reads the activations under a zero trit (inference.c:128): a caller may hand in a 256-byte row for
    // n_input = 260.  Read exactly what the reference can read: up to the last non-zero trit of any row.
    uint32_t valid_in = n_input;
    if (enc == BNM_ENC_TERNARY) {
        const uint16_t *w16 = reinterpret_cast<const uint16_t *>(weights);
        const uint32_t wpr = n_input / 10;
        valid_in = 0;
        for (uint32_t o = 0; o < n_output; o++)
            for (uint32_t g = wpr; g-- > 0;) {
                if (g * 10 + 10 <= valid_in) break;
                uint32_t c = w16[(size_t)o * wpr + g];
                for (uint32_t j = 0; j < 10; j++) {
                    c *= 3u;
                    if (!(c & 0x20000u)) valid_in = std::max(valid_in, g * 10 + j + 1);
                    c &= 0xFFFFu;
                }
            }
    }
    return host_call([&](HostStaging &s) {
        const size_t need = packed_weight_bytes(enc, n_input, n_output);
        uint8_t *packed;
        CU_TRY(s.get(&packed, need + 16));
        CU_TRY(cudaMemsetAsync(packed, 0, need + 16, s.st));
        if (need) CU_TRY(cudaMemcpyAsync(packed, weights, need, cudaMemcpyHostToDevice, s.st));
        FcLayerDev L;
        if (cudaError_t e = decode_fc_layer(packed, enc, n_input, n_output, nf4_extension, L, s.pool, s.st))
            return fail(BNM_E_CUDA, "weight decode of an FC layer failed: %s", cudaGetErrorString(e));
        struct Planes { FcLayerDev &L; cudaStream_t st; ~Planes() { free_fc_layer(L, st); } } planes{L, s.st};   // on every return below
        int8_t *act;
        int32_t *out;
        CU_TRY(s.get(&act, n * (size_t)L.k_pad));
        CU_TRY(s.out(&out, output, n * (size_t)n_output));
        CU_TRY(cudaMemsetAsync(act, 0, n * (size_t)L.k_pad, s.st));
        if (valid_in) CU_TRY(cudaMemcpy2DAsync(act, L.k_pad, activations, n_input, valid_in, n, cudaMemcpyHostToDevice, s.st));
        if (!launch_fc_dp4a(act, L.k_pad, L, out, n, s.st))
            return fail(BNM_E_UNSUPPORTED, "processfclayer: n_input %u needs more shared memory than an SM has (layer kernel stages 128 rows)", n_input);
        return 0;
    });
}

extern "C" int bnm_relunorm_batch(const int32_t *input, int8_t *output, uint32_t *argmax, uint32_t n_input, size_t n) {
    if (int rc = require_device()) return rc;
    if (n == 0) return 0;
    if (n_input == 0) {   // inference.c:24-37: nothing is scanned, position stays 255
        if (argmax) for (size_t i = 0; i < n; i++) argmax[i] = 255;
        return 0;
    }
    if (!input) return fail(BNM_E_ARG, "bnm_relunorm_batch: null input");
    return host_call([&](HostStaging &s) {
        int32_t *in;
        uint32_t *am;
        int8_t *out;
        CU_TRY(s.in(&in, input, n * (size_t)n_input));   // copied in before anything is copied out: output may alias input
        CU_TRY(s.out(&am, argmax, n));
        CU_TRY(s.out(&out, output, output ? n * (size_t)n_input : 0));
        launch_relunorm(in, n_input, out, n_input, am, n, s.st);
        return 0;
    });
}

extern "C" int bnm_conv33relu_batch(const int32_t *activations, const int8_t *weights, uint32_t n_w, uint32_t xy, uint32_t n_shift,
                                    int32_t *output, size_t n) {
    if (int rc = require_device()) return rc;
    if (n == 0 || xy < 3) return 0;
    if (!activations || !weights || !output || n_w == 0) return fail(BNM_E_ARG, "bnm_conv33relu_batch: null argument");
    return host_call([&](HostStaging &s) {
        int32_t *in, *out;
        int8_t *w;
        CU_TRY(s.in(&in, activations, n * (size_t)xy * xy));
        CU_TRY(s.in(&w, weights, (size_t)n_w * 9));
        CU_TRY(s.out(&out, output, n * (size_t)(xy - 2) * (xy - 2)));
        launch_conv33relu(in, w, n_w, xy, n_shift, out, n, s.st);
        return 0;
    });
}

extern "C" int bnm_maxpool22_batch(const int32_t *activations, uint32_t xy, int32_t *output, size_t n) {
    if (int rc = require_device()) return rc;
    if (n == 0 || xy < 2) return 0;
    if (!activations || !output) return fail(BNM_E_ARG, "bnm_maxpool22_batch: null argument");
    return host_call([&](HostStaging &s) {
        int32_t *in, *out;
        CU_TRY(s.in(&in, activations, n * (size_t)xy * xy));
        CU_TRY(s.out(&out, output, n * (size_t)(xy / 2) * (xy / 2)));
        launch_maxpool22(in, xy, out, n, s.st);
        return 0;
    });
}

extern "C" int bnm_quantize_images_device(const float *images, size_t n, uint32_t elems, int8_t *out, void *stream) {
    if (int rc = require_device()) return rc;
    if (n == 0 || elems == 0) return 0;
    if (!images || !out) return fail(BNM_E_ARG, "bnm_quantize_images_device: null argument");
    launch_quantize_images(images, elems, out, n, static_cast<cudaStream_t>(stream));
    return launch_status();
}

extern "C" int bnm_quantize_images_device_f16(const uint16_t *images, int format, size_t n, uint32_t elems, int8_t *out, void *stream) {
    if (int rc = require_device()) return rc;
    if (format != BNM_FLOAT16 && format != BNM_BFLOAT16)
        return fail(BNM_E_ARG, "bnm_quantize_images_device_f16: format %d, must be BNM_FLOAT16 (1) or BNM_BFLOAT16 (2)", format);
    if (n == 0 || elems == 0) return 0;
    if (!images || !out) return fail(BNM_E_ARG, "bnm_quantize_images_device_f16: null argument");
    launch_quantize_images(images, static_cast<HalfFormat>(format), elems, out, n, static_cast<cudaStream_t>(stream));
    return launch_status();
}

extern "C" int bnm_quantize_images(const float *images, size_t n, uint32_t elems, int8_t *out) {
    if (int rc = require_device()) return rc;
    if (n == 0 || elems == 0) return 0;
    if (!images || !out) return fail(BNM_E_ARG, "bnm_quantize_images: null argument");
    return host_call([&](HostStaging &s) {
        float *in;
        int8_t *q;
        CU_TRY(s.in(&in, images, n * (size_t)elems));
        CU_TRY(s.out(&q, out, n * (size_t)elems));
        launch_quantize_images(in, elems, q, n, s.st);
        return 0;
    });
}

// -----------------------------------------------------------------------------------------------
// Emulation mode (SURVEY.md 8f rank 4): QuantizedModel.inference_quantized of the reference (BitNetMCU.py:420-535) on the GPU --
// float images in, float64 "logits" out, with the EMULATOR's normalisation rules (power-of-two rescale to max <= 127 with
// round-half-even for BitLinear, per-image renormalisation of every conv output) instead of the C engine's.  It reuses the
// engine's integer kernels (decoded weights, dp4a layers, conv / pool); weight levels are the engine's integers divided by
// level_scale (2 for 2bitsym / 4bitsym), so every intermediate is an exact dyadic rational and the result equals NumPy's.
// On the fused path (fc_wgmma.cu):
//   * FC models whose rows have <= 256 elements, up to 64 wide with <= 16 classes: one kernel, fc_emul_kernel;
//   * other FC models: the scaling kernel (k_quantize_images), then fc_emul_i8_kernel at the plan's width;
//   * CNN models up to kCnnEmulMaxChannels channels: the front-end kernel k_cnn_emul_frontend, then fc_emul_i8_kernel on its features;
//     the window scan runs k_quantize_windows, then the same front-end on the scaled rows (k_cnn_emul_frontend_i8).
// BNM_PATH_LAYERS, models without a fused plan and wider CNN models run the emulation kernels layer by layer (choose_route).
// -----------------------------------------------------------------------------------------------
int bnm::level_shift_of(int32_t enc) { return (enc == BNM_ENC_2BITSYM || enc == BNM_ENC_4BITSYM) ? 1 : 0; }

// -----------------------------------------------------------------------------------------------
// Both engines in one call (test_inference.py:130-175): the C engine's and the emulator's labels of the same float images, and
// counts of their agreement and of their accuracy against truth.  The one-pass kernel where both float-input rows exist; every
// other model runs the C engine's float route and the emulator's route per pass, into the caller's label buffers or the call's
// scratch, then k_engine_counts (run_engines).
// -----------------------------------------------------------------------------------------------
// the two engines' route r without a fused form on n float images (of r's input kind) on st (capture state cap) -> out: labels
// (the C engine's) and engines
static int run_engines(bnm_model *m, const Route &r, const void *images, size_t n, const FcOutputs &out, cudaStream_t st,
                       const StreamCapture &cap) {
    const EngineOutputs &e = out.engines;
    const Route c_route = choose_route(m, kEngineC, r.in, false), py_route = choose_route(m, kEngineEmul, r.in, false);
    const size_t chunk = std::min(n, r.pass), row_bytes = m->img_bytes * in_elem_bytes(r.in);
    Scratch scratch(m->pool, st);
    uint32_t *own[2];   // C / emulator labels the caller does not take
    CU_TRY(scratch.get(&own[0], e.counts && !out.labels ? chunk : 0));
    CU_TRY(scratch.get(&own[1], e.counts && !e.labels_py ? chunk : 0));
    for (size_t b = 0; b < n; b += chunk) {
        const size_t nb = std::min(chunk, n - b);
        const void *img = static_cast<const char *>(images) + b * row_bytes;
        uint32_t *lc = out.labels ? out.labels + b : own[0];
        uint32_t *lp = e.labels_py ? e.labels_py + b : own[1];
        if (lc)
            if (int rc = run_route(m, c_route, img, nb, FcOutputs{nullptr, lc}, st, cap)) return rc;
        if (lp)
            if (int rc = run_route(m, py_route, img, nb, FcOutputs{nullptr, lp}, st, cap)) return rc;
        if (e.counts) launch_engine_counts(lc, lp, e.truth ? e.truth + b : nullptr, nb, m->n_classes, e.counts, st);
    }
    return launch_status();
}

// -----------------------------------------------------------------------------------------------
// the inference entries: each fills one call record, which run_call checks (check_call) and runs
// -----------------------------------------------------------------------------------------------
// One inference entry's call: the arguments of choose_route, the input, the outputs, and the rules in which entries differ.  A top-k
// call needs classes when n > 0, checks k and its buffers' alignment whatever n, and names its route under BNM_VERBOSE.
struct Call {
    const char *name;   // the entry, for messages
    Engine engine;
    InKind in;
    bool topk;          // the k best classes out
    const void *images;
    size_t n;
    FcOutputs out;      // the two engines' entry: the C engine's labels in labels, the rest in engines
    struct { size_t images = 1, logits = 1, classes = 1, scores = 1, counts = 1; } align;   // in bytes; labels and truth: any
    void *stream = nullptr;        // a device entry's stream
    bool host = false;             // host buffers: a synchronous call through the small-batch path or the host pipeline
    bool need_logits = false;      // logits must be given when n > 0 (the emulator's host entry)
    bool no_output_at_0 = false;   // a call without outputs is an error even when n == 0 (the two engines' entry)
    const WindowGrid *windows = nullptr;   // the window scan: the images are the n windows of this grid, `images` its first plane
};

// The argument rules, in this order: a null model, or (n > 0) null images, classes or needed logits; no output at all; k out of
// range; a misaligned buffer.  n == 0 ends the checks before the alignment ones except on a top-k call.
static int check_call(const bnm_model *m, const Call &c) {
    const FcOutputs &o = c.out;
    if (!m || (c.n && (!c.images || (c.topk && !o.topk.classes) || (c.need_logits && !o.logits))))
        return fail(BNM_E_ARG, "%s: null argument", c.name);
    const bool output = o.logits || o.labels || (o.gather && (o.gather->n_labels_dst || o.gather->n_logits_dst)) || o.topk.classes ||
                        o.engines.labels_py || o.engines.counts;
    if (!output && (c.n || c.no_output_at_0)) return fail(BNM_E_ARG, "%s: no output (every output buffer NULL)", c.name);
    if (c.topk && (o.topk.k < 1 || o.topk.k > std::min<uint32_t>(m->n_classes, BNM_MAX_TOPK)))
        return fail(BNM_E_ARG, "%s: k = %u, must be 1 .. min(n_classes = %u, %d)", c.name, o.topk.k, m->n_classes, BNM_MAX_TOPK);
    if (!c.n && !c.topk) return 0;
    const struct { const void *p; size_t align; const char *what; } bufs[] = {
        {c.images, c.align.images, "device image buffer"}, {o.logits, c.align.logits, "device logits buffer"},
        {o.topk.classes, c.align.classes, "classes buffer"}, {o.topk.scores, c.align.scores, "scores buffer"},
        {o.engines.counts, c.align.counts, "device counts"}};
    for (const auto &b : bufs)
        if ((uintptr_t)b.p & (b.align - 1)) return fail(BNM_E_ARG, "%s: the %s must be %zu-byte aligned", c.name, b.what, b.align);
    return 0;
}

// Check call c and run its route: on the device entry's stream, whose capture state it reads once; for the two engines without a
// fused form, run_engines; the C engine's int8 host calls of up to kSmallBatch images (and chunk) through infer_small, every other
// host call through infer_pipelined.
static int run_call(bnm_model *m, const Call &c) {
    if (int rc = check_call(m, c)) return rc;
    if (c.n == 0) return 0;
    const FcOutputs &o = c.out;
    if (c.host && c.engine == kEngineC && !c.topk && !c.windows && c.n <= kSmallBatch && c.n <= m->chunk_images)   // sets the device where it launches
        return infer_small(m, static_cast<const int8_t *>(c.images), c.n, static_cast<int32_t *>(o.logits), o.labels);
    CU_TRY(cudaSetDevice(m->device));
    const Route r = choose_route(m, c.engine, c.in, c.topk, c.windows);
    // the lines of the model's creation name the float32 routes only: a 16-bit call names its own (a 16-bit form or scaling kernel);
    // a host window scan names its route with its bands (infer_pipelined)
    if ((c.topk || c.windows || half_in(c.in)) && m->verbose && !(c.host && c.windows))
        print_route(m, (std::string(c.windows ? "windows route: " : c.topk ? "topk route: " : "16-bit route: ") + c.name).c_str(), r);
    if (o.gather && !r.fused)
        return fail(BNM_E_UNSUPPORTED, "the fused result exchange needs the fused tensor-core path (model: %s)", m->plan_err.c_str());
    cudaStream_t st = static_cast<cudaStream_t>(c.stream);
    if (c.host) return infer_pipelined(m, r, c.images, c.n, o, c.windows, c.name);
    const StreamCapture cap = capture_of(st);
    if (c.engine == kEngineBoth && !r.fused) return run_engines(m, r, c.images, c.n, o, st, cap);
    return run_route(m, r, c.images, c.n, o, st, cap, c.windows);
}

extern "C" int bnm_infer_batch_device_gather(bnm_model *m, const int8_t *images, size_t n, int32_t *logits, uint32_t *labels,
                                             const bnm_gather *gather, void *stream) {
    static_assert(sizeof(bnm_gather) == sizeof(GatherDst), "bnm_gather and GatherDst must share their layout");
    if (gather && (gather->n_labels_dst > BNM_MAX_GATHER_DST || gather->n_logits_dst > BNM_MAX_GATHER_DST))
        return fail(BNM_E_ARG, "at most %d gather destinations", BNM_MAX_GATHER_DST);
    if (gather)
        for (uint32_t d = 0; d < gather->n_logits_dst; d++)
            if ((uintptr_t)gather->logits_dst[d] & 7) return fail(BNM_E_ARG, "gather logits buffers must be 8-byte aligned");
    const GatherDst *g = reinterpret_cast<const GatherDst *>(gather);
    return run_call(m, {"bnm_infer_batch_device", kEngineC, kInI8, false, images, n, {logits, labels, g}, {16, 8}, stream});
}

extern "C" int bnm_infer_batch_device(bnm_model *m, const int8_t *images, size_t n, int32_t *logits, uint32_t *labels, void *stream) {
    return bnm_infer_batch_device_gather(m, images, n, logits, labels, nullptr, stream);
}

// float images -> logits / labels on the device.  FC models on the fused path (rows of <= 256 elements, <= 16 classes): ONE kernel, the
// input scaling fused into its load stage.  Everything else: per pass of 2^20 images the scaling kernel into the call's scratch,
// then the int8 route on it.
extern "C" int bnm_infer_batch_device_f32(bnm_model *m, const float *images, size_t n, int32_t *logits, uint32_t *labels, void *stream) {
    return run_call(m, {"bnm_infer_batch_device_f32", kEngineC, kInF32, false, images, n, {logits, labels}, {16, 8}, stream});
}

extern "C" int bnm_emulate_batch_device(bnm_model *m, const float *images, size_t n, double *logits, uint32_t *labels, void *stream) {
    return run_call(m, {"bnm_emulate_batch_device", kEngineEmul, kInF32, false, images, n, {logits, labels}, {16, 8}, stream});
}

extern "C" int bnm_compare_engines_device(bnm_model *m, const float *images, size_t n, const uint32_t *truth, uint32_t *labels_c,
                                          uint32_t *labels_py, bnm_engine_counts *counts, void *stream) {
    static_assert(sizeof(bnm_engine_counts) == 4 * sizeof(unsigned long long), "bnm_engine_counts: four 64-bit counters");
    if (truth && !counts) return fail(BNM_E_ARG, "bnm_compare_engines_device: truth without counts");
    const FcOutputs out{nullptr, labels_c, nullptr, {}, {labels_py, truth, reinterpret_cast<unsigned long long *>(counts)}};
    return run_call(m, {"bnm_compare_engines_device", kEngineBoth, kInF32, false, images, n, out, {16, 1, 1, 1, 8}, stream, false, false,
                        true});   // no outputs: an error even at n == 0
}

// Top-k (section 8): the k best classes of every image and their scores -- the classes ranked by logit, highest first, ties to the
// lower class, so rank 0 is the label of the matching entry -- and no logits written anywhere.
//   * FC models on the fused path: one launch of fc_topk_kernel, whose epilogue ranks the classes in registers;
//   * CNN models on the fused path: the front-end into the feature scratch, then that kernel, in chunks of 2^20 images;
//   * BNM_PATH_LAYERS and models without a fused plan: the layer-by-layer chain into its int32 scratch (the emulator: its float64
//     logits into a chunk of scratch), then k_topk_rows.
// The float entry scales each pass of 2^20 images into its own scratch, then runs the int8 route on it; the emulator runs its own
// front-end (scaling kernel or CNN front-end) into its scratch, then fc_topk_kernel with its rule.  choose_route picks the route.
extern "C" int bnm_infer_topk_device(bnm_model *m, const int8_t *images, size_t n, uint32_t k, uint32_t *classes, int32_t *scores, void *stream) {
    return run_call(m, {"bnm_infer_topk_device", kEngineC, kInI8, true, images, n, {nullptr, nullptr, nullptr, {k, classes, scores}}, {16, 1, 4, 4}, stream});
}

extern "C" int bnm_infer_topk_device_f32(bnm_model *m, const float *images, size_t n, uint32_t k, uint32_t *classes, int32_t *scores, void *stream) {
    return run_call(m, {"bnm_infer_topk_device_f32", kEngineC, kInF32, true, images, n, {nullptr, nullptr, nullptr, {k, classes, scores}}, {16, 1, 4, 4}, stream});
}

extern "C" int bnm_emulate_topk_device(bnm_model *m, const float *images, size_t n, uint32_t k, uint32_t *classes, double *scores, void *stream) {
    return run_call(m, {"bnm_emulate_topk_device", kEngineEmul, kInF32, true, images, n, {nullptr, nullptr, nullptr, {k, classes, scores}}, {16, 1, 4, 8}, stream});
}

// Window scan (sections 9, 10, 12 and 13): every 16x16 window of a stack of float32 or 16-bit planes, padded or not, on a stride
// grid, classified as the entry named in the header classifies the extracted windows (widened to float32, padded as
// torch.nn.functional.pad pads).  Per pass of 2^20 windows (the layered emulator: of its own pass), k_quantize_windows scales them
// from the planes into the call's scratch, then that entry's route runs on the scaled rows; a fused FC launch after it keeps its
// wait and counts as a launch of another kind.  w's checks and pad's (NULL: no padding, the grid of sections 9 to 12), then call c
// (name, engine, the planes' element kind, top-k, outputs, alignment, stream) on its windows.  Windows: bnm_windows or
// bnm_windows_f16, whose fields differ in the image's element type only, or (a host call, section 14) bnm_windows_host, whose
// rows and planes may be any number of elements apart.
template <class Windows> static int run_windows(bnm_model *m, const Windows *w, Call c, const bnm_window_padding *pad = nullptr) {
    if (int rc = require_device()) return rc;
    if (!w) return fail(BNM_E_ARG, "%s: null window descriptor", c.name);
    if (!w->stride_y || !w->stride_x) return fail(BNM_E_ARG, "%s: zero stride (%u, %u)", c.name, w->stride_y, w->stride_x);
    const size_t row_elems = c.host ? 1 : 16 / in_elem_bytes(c.in);   // elements in 16 bytes: a device page's row and plane alignment
    if (c.host && w->pitch < w->width) return fail(BNM_E_ARG, "%s: pitch %zu must be >= width %u", c.name, w->pitch, w->width);
    if (w->pitch < w->width || w->pitch % row_elems)
        return fail(BNM_E_ARG, "%s: pitch %zu must be >= width %u and a multiple of %zu elements (16-byte rows)", c.name, w->pitch,
                    w->width, row_elems);
    if (w->planes > 1 && w->plane_pitch % row_elems)
        return fail(BNM_E_ARG, "%s: plane pitch %zu must be a multiple of %zu elements (16-byte aligned planes)", c.name,
                    w->plane_pitch, row_elems);
    if (m && m->img_bytes != 256)
        return fail(BNM_E_UNSUPPORTED, "%s: windows are 16x16 images, the model takes %u-element images", c.name, m->img_bytes);
    const bnm_window_padding none{};
    const bnm_window_padding &pd = pad ? *pad : none;
    if (pad) {
        if (pd.left > 15 || pd.right > 15 || pd.top > 15 || pd.bottom > 15)
            return fail(BNM_E_ARG, "%s: padding (left %u, right %u, top %u, bottom %u): each side must be at most 15", c.name, pd.left,
                        pd.right, pd.top, pd.bottom);
        if (pd.mode != BNM_PAD_CONSTANT && pd.mode != BNM_PAD_REPLICATE && pd.mode != BNM_PAD_REFLECT)
            return fail(BNM_E_ARG, "%s: padding mode %u, must be BNM_PAD_CONSTANT (0), BNM_PAD_REPLICATE (1) or BNM_PAD_REFLECT (2)",
                        c.name, pd.mode);
        const bool empty = !w->planes || !w->height || !w->width;   // no windows, whatever the padding
        if (!empty && pd.mode == BNM_PAD_REFLECT && (pd.top >= w->height || pd.bottom >= w->height || pd.left >= w->width || pd.right >= w->width))
            return fail(BNM_E_ARG, "%s: reflect padding (left %u, right %u, top %u, bottom %u) must be less than the page's %u x %u on each side",
                        c.name, pd.left, pd.right, pd.top, pd.bottom, w->height, w->width);
    }
    // the grid over the padded planes, sized in 64 bits; a page of no pixels has no windows, padded or not
    const uint64_t pad_h = (uint64_t)w->height + pd.top + pd.bottom, pad_w = (uint64_t)w->width + pd.left + pd.right;
    if (pad_h > UINT32_MAX || pad_w > UINT32_MAX)
        return fail(BNM_E_ARG, "%s: the padded page (%llu x %llu) must be at most 2^32 - 1 pixels either way", c.name,
                    (unsigned long long)pad_h, (unsigned long long)pad_w);
    const uint32_t out_h = pad_h < 16 ? 0 : (uint32_t)((pad_h - 16) / w->stride_y + 1);
    const uint32_t out_w = pad_w < 16 ? 0 : (uint32_t)((pad_w - 16) / w->stride_x + 1);
    const WindowGrid g{w->image, half_in(c.in) ? (uint32_t)half_format(c.in) : 0u, w->planes, w->height, w->width, w->pitch,
                       w->planes > 1 ? w->plane_pitch : 0, w->stride_y, w->stride_x, out_h, out_w,
                       pd.top, pd.left, pd.right, pd.mode, pd.value};
    c.images = w->image;
    c.n = w->height && w->width ? (size_t)w->planes * out_h * out_w : 0;
    c.windows = &g;
    return run_call(m, c);
}

extern "C" int bnm_infer_windows_device_f32(bnm_model *m, const float *image, uint32_t height, uint32_t width, size_t pitch,
                                            uint32_t stride_y, uint32_t stride_x, int32_t *logits, uint32_t *labels, void *stream) {
    const bnm_windows w{image, 1, height, width, pitch, 0, stride_y, stride_x};
    return run_windows(m, &w, {"bnm_infer_windows_device_f32", kEngineC, kInF32, false, image, 0, {logits, labels}, {16, 8}, stream});
}

extern "C" int bnm_scan_windows_device(bnm_model *m, const bnm_windows *w, int32_t *logits, uint32_t *labels, void *stream) {
    return run_windows(m, w, {"bnm_scan_windows_device", kEngineC, kInF32, false, nullptr, 0, {logits, labels}, {16, 8}, stream});
}

extern "C" int bnm_scan_windows_topk_device(bnm_model *m, const bnm_windows *w, uint32_t k, uint32_t *classes, int32_t *scores,
                                            void *stream) {
    return run_windows(m, w, {"bnm_scan_windows_topk_device", kEngineC, kInF32, true, nullptr, 0, {nullptr, nullptr, nullptr, {k, classes, scores}},
                              {16, 1, 4, 4}, stream});
}

extern "C" int bnm_emulate_windows_device(bnm_model *m, const bnm_windows *w, double *logits, uint32_t *labels, void *stream) {
    return run_windows(m, w, {"bnm_emulate_windows_device", kEngineEmul, kInF32, false, nullptr, 0, {logits, labels}, {16, 8}, stream});
}

extern "C" int bnm_emulate_windows_topk_device(bnm_model *m, const bnm_windows *w, uint32_t k, uint32_t *classes, double *scores,
                                               void *stream) {
    return run_windows(m, w, {"bnm_emulate_windows_topk_device", kEngineEmul, kInF32, true, nullptr, 0,
                              {nullptr, nullptr, nullptr, {k, classes, scores}}, {16, 1, 4, 8}, stream});
}

// 16-bit float images (section 11): call c of the float32 sibling, its input kind the one of `format` (BNM_E_ARG for any other
// value, whatever n).  Its route is the sibling's (choose_route) and every output is the sibling's on the images widened to float32.
static int half_kind(const char *name, int format, InKind &in) {
    if (format != BNM_FLOAT16 && format != BNM_BFLOAT16)
        return fail(BNM_E_ARG, "%s: format %d, must be BNM_FLOAT16 (1) or BNM_BFLOAT16 (2)", name, format);
    in = format == BNM_BFLOAT16 ? kInBF16 : kInF16;
    return 0;
}
static int run_half(bnm_model *m, int format, Call c) {
    if (int rc = half_kind(c.name, format, c.in)) return rc;
    return run_call(m, c);
}

extern "C" int bnm_infer_batch_device_f16(bnm_model *m, const uint16_t *images, int format, size_t n, int32_t *logits, uint32_t *labels,
                                          void *stream) {
    return run_half(m, format, {"bnm_infer_batch_device_f16", kEngineC, kInF16, false, images, n, {logits, labels}, {16, 8}, stream});
}

extern "C" int bnm_emulate_batch_device_f16(bnm_model *m, const uint16_t *images, int format, size_t n, double *logits, uint32_t *labels,
                                            void *stream) {
    return run_half(m, format, {"bnm_emulate_batch_device_f16", kEngineEmul, kInF16, false, images, n, {logits, labels}, {16, 8}, stream});
}

extern "C" int bnm_compare_engines_device_f16(bnm_model *m, const uint16_t *images, int format, size_t n, const uint32_t *truth,
                                              uint32_t *labels_c, uint32_t *labels_py, bnm_engine_counts *counts, void *stream) {
    if (truth && !counts) return fail(BNM_E_ARG, "bnm_compare_engines_device_f16: truth without counts");
    const FcOutputs out{nullptr, labels_c, nullptr, {}, {labels_py, truth, reinterpret_cast<unsigned long long *>(counts)}};
    return run_half(m, format, {"bnm_compare_engines_device_f16", kEngineBoth, kInF16, false, images, n, out, {16, 1, 1, 1, 8}, stream,
                                false, false, true});   // no outputs: an error even at n == 0
}

extern "C" int bnm_infer_topk_device_f16(bnm_model *m, const uint16_t *images, int format, size_t n, uint32_t k, uint32_t *classes,
                                         int32_t *scores, void *stream) {
    return run_half(m, format, {"bnm_infer_topk_device_f16", kEngineC, kInF16, true, images, n, {nullptr, nullptr, nullptr, {k, classes, scores}},
                                {16, 1, 4, 4}, stream});
}

extern "C" int bnm_emulate_topk_device_f16(bnm_model *m, const uint16_t *images, int format, size_t n, uint32_t k, uint32_t *classes,
                                           double *scores, void *stream) {
    return run_half(m, format, {"bnm_emulate_topk_device_f16", kEngineEmul, kInF16, true, images, n, {nullptr, nullptr, nullptr, {k, classes, scores}},
                                {16, 1, 4, 8}, stream});
}

// 16-bit pages (section 12): the stacked window entries of section 10 on a bnm_windows_f16, which one Python structure serves with
// bnm_windows; the planes' element kind is the one of `format`, and every output is the sibling's on the planes widened to float32
static_assert(sizeof(bnm_windows_f16) == sizeof(bnm_windows) && offsetof(bnm_windows_f16, image) == offsetof(bnm_windows, image) &&
                  offsetof(bnm_windows_f16, planes) == offsetof(bnm_windows, planes) &&
                  offsetof(bnm_windows_f16, height) == offsetof(bnm_windows, height) &&
                  offsetof(bnm_windows_f16, width) == offsetof(bnm_windows, width) &&
                  offsetof(bnm_windows_f16, pitch) == offsetof(bnm_windows, pitch) &&
                  offsetof(bnm_windows_f16, plane_pitch) == offsetof(bnm_windows, plane_pitch) &&
                  offsetof(bnm_windows_f16, stride_y) == offsetof(bnm_windows, stride_y) &&
                  offsetof(bnm_windows_f16, stride_x) == offsetof(bnm_windows, stride_x),
              "bnm_windows_f16 has the field layout of bnm_windows");
static int run_windows_half(bnm_model *m, const bnm_windows_f16 *w, int format, Call c) {
    if (int rc = half_kind(c.name, format, c.in)) return rc;
    return run_windows(m, w, c);
}

extern "C" int bnm_scan_windows_device_f16(bnm_model *m, const bnm_windows_f16 *w, int format, int32_t *logits, uint32_t *labels,
                                           void *stream) {
    return run_windows_half(m, w, format, {"bnm_scan_windows_device_f16", kEngineC, kInF16, false, nullptr, 0, {logits, labels}, {16, 8}, stream});
}

extern "C" int bnm_scan_windows_topk_device_f16(bnm_model *m, const bnm_windows_f16 *w, int format, uint32_t k, uint32_t *classes,
                                                int32_t *scores, void *stream) {
    return run_windows_half(m, w, format, {"bnm_scan_windows_topk_device_f16", kEngineC, kInF16, true, nullptr, 0,
                                           {nullptr, nullptr, nullptr, {k, classes, scores}}, {16, 1, 4, 4}, stream});
}

extern "C" int bnm_emulate_windows_device_f16(bnm_model *m, const bnm_windows_f16 *w, int format, double *logits, uint32_t *labels,
                                              void *stream) {
    return run_windows_half(m, w, format, {"bnm_emulate_windows_device_f16", kEngineEmul, kInF16, false, nullptr, 0, {logits, labels}, {16, 8},
                                           stream});
}

extern "C" int bnm_emulate_windows_topk_device_f16(bnm_model *m, const bnm_windows_f16 *w, int format, uint32_t k, uint32_t *classes,
                                                   double *scores, void *stream) {
    return run_windows_half(m, w, format, {"bnm_emulate_windows_topk_device_f16", kEngineEmul, kInF16, true, nullptr, 0,
                                           {nullptr, nullptr, nullptr, {k, classes, scores}}, {16, 1, 4, 8}, stream});
}

// Padded pages (section 13): the stacked window entries of sections 10 and 12 on the planes padded as torch.nn.functional.pad pads
// them (BNM_E_ARG for a NULL padding); the same Call as the sibling's, and k_quantize_windows makes the border as it loads a band
static_assert(BNM_PAD_CONSTANT == kPadConstant && BNM_PAD_REPLICATE == kPadReplicate && BNM_PAD_REFLECT == kPadReflect,
              "BNM_PAD_* are the kernel's PadMode values");
template <class Windows> static int run_windows_padded(bnm_model *m, const Windows *w, const bnm_window_padding *pad, Call c) {
    if (!pad) return fail(BNM_E_ARG, "%s: null padding", c.name);
    return run_windows(m, w, c, pad);
}
static int run_windows_padded_half(bnm_model *m, const bnm_windows_f16 *w, int format, const bnm_window_padding *pad, Call c) {
    if (int rc = half_kind(c.name, format, c.in)) return rc;
    return run_windows_padded(m, w, pad, c);
}

extern "C" int bnm_scan_windows_padded_device(bnm_model *m, const bnm_windows *w, const bnm_window_padding *padding, int32_t *logits,
                                              uint32_t *labels, void *stream) {
    return run_windows_padded(m, w, padding, {"bnm_scan_windows_padded_device", kEngineC, kInF32, false, nullptr, 0, {logits, labels}, {16, 8}, stream});
}

extern "C" int bnm_scan_windows_topk_padded_device(bnm_model *m, const bnm_windows *w, const bnm_window_padding *padding, uint32_t k,
                                                   uint32_t *classes, int32_t *scores, void *stream) {
    return run_windows_padded(m, w, padding, {"bnm_scan_windows_topk_padded_device", kEngineC, kInF32, true, nullptr, 0,
                                              {nullptr, nullptr, nullptr, {k, classes, scores}}, {16, 1, 4, 4}, stream});
}

extern "C" int bnm_emulate_windows_padded_device(bnm_model *m, const bnm_windows *w, const bnm_window_padding *padding, double *logits,
                                                 uint32_t *labels, void *stream) {
    return run_windows_padded(m, w, padding, {"bnm_emulate_windows_padded_device", kEngineEmul, kInF32, false, nullptr, 0, {logits, labels},
                                              {16, 8}, stream});
}

extern "C" int bnm_emulate_windows_topk_padded_device(bnm_model *m, const bnm_windows *w, const bnm_window_padding *padding, uint32_t k,
                                                      uint32_t *classes, double *scores, void *stream) {
    return run_windows_padded(m, w, padding, {"bnm_emulate_windows_topk_padded_device", kEngineEmul, kInF32, true, nullptr, 0,
                                              {nullptr, nullptr, nullptr, {k, classes, scores}}, {16, 1, 4, 8}, stream});
}

extern "C" int bnm_scan_windows_padded_device_f16(bnm_model *m, const bnm_windows_f16 *w, int format, const bnm_window_padding *padding,
                                                  int32_t *logits, uint32_t *labels, void *stream) {
    return run_windows_padded_half(m, w, format, padding, {"bnm_scan_windows_padded_device_f16", kEngineC, kInF16, false, nullptr, 0,
                                                           {logits, labels}, {16, 8}, stream});
}

extern "C" int bnm_scan_windows_topk_padded_device_f16(bnm_model *m, const bnm_windows_f16 *w, int format, const bnm_window_padding *padding,
                                                       uint32_t k, uint32_t *classes, int32_t *scores, void *stream) {
    return run_windows_padded_half(m, w, format, padding, {"bnm_scan_windows_topk_padded_device_f16", kEngineC, kInF16, true, nullptr, 0,
                                                           {nullptr, nullptr, nullptr, {k, classes, scores}}, {16, 1, 4, 4}, stream});
}

extern "C" int bnm_emulate_windows_padded_device_f16(bnm_model *m, const bnm_windows_f16 *w, int format, const bnm_window_padding *padding,
                                                     double *logits, uint32_t *labels, void *stream) {
    return run_windows_padded_half(m, w, format, padding, {"bnm_emulate_windows_padded_device_f16", kEngineEmul, kInF16, false, nullptr, 0,
                                                           {logits, labels}, {16, 8}, stream});
}

extern "C" int bnm_emulate_windows_topk_padded_device_f16(bnm_model *m, const bnm_windows_f16 *w, int format,
                                                          const bnm_window_padding *padding, uint32_t k, uint32_t *classes, double *scores,
                                                          void *stream) {
    return run_windows_padded_half(m, w, format, padding, {"bnm_emulate_windows_topk_padded_device_f16", kEngineEmul, kInF16, true, nullptr,
                                                           0, {nullptr, nullptr, nullptr, {k, classes, scores}}, {16, 1, 4, 8}, stream});
}

// Host pages (section 14): the stacked window entries on a stack in host memory, padded or not (pad NULL), in the element kind of
// its format; call c of the device sibling with host buffers, run by infer_pipelined band by band
static int run_windows_host(bnm_model *m, const bnm_windows_host *w, const bnm_window_padding *pad, Call c) {
    if (int rc = require_device()) return rc;
    if (!w) return fail(BNM_E_ARG, "%s: null window descriptor", c.name);
    if (w->format != BNM_FLOAT32 && w->format != BNM_FLOAT16 && w->format != BNM_BFLOAT16)
        return fail(BNM_E_ARG, "%s: format %d, must be BNM_FLOAT32 (3), BNM_FLOAT16 (1) or BNM_BFLOAT16 (2)", c.name, w->format);
    c.in = w->format == BNM_FLOAT32 ? kInF32 : w->format == BNM_BFLOAT16 ? kInBF16 : kInF16;
    return run_windows(m, w, c, pad);
}

extern "C" int bnm_scan_windows(bnm_model *m, const bnm_windows_host *w, const bnm_window_padding *padding, int32_t *logits,
                                uint32_t *labels) {
    return run_windows_host(m, w, padding, {"bnm_scan_windows", kEngineC, kInF32, false, nullptr, 0, {logits, labels}, {}, nullptr, true});
}

extern "C" int bnm_scan_windows_topk(bnm_model *m, const bnm_windows_host *w, const bnm_window_padding *padding, uint32_t k,
                                     uint32_t *classes, int32_t *scores) {
    return run_windows_host(m, w, padding, {"bnm_scan_windows_topk", kEngineC, kInF32, true, nullptr, 0,
                                            {nullptr, nullptr, nullptr, {k, classes, scores}}, {}, nullptr, true});
}

extern "C" int bnm_emulate_windows(bnm_model *m, const bnm_windows_host *w, const bnm_window_padding *padding, double *logits,
                                   uint32_t *labels) {
    return run_windows_host(m, w, padding, {"bnm_emulate_windows", kEngineEmul, kInF32, false, nullptr, 0, {logits, labels}, {}, nullptr,
                                            true});
}

extern "C" int bnm_emulate_windows_topk(bnm_model *m, const bnm_windows_host *w, const bnm_window_padding *padding, uint32_t k,
                                        uint32_t *classes, double *scores) {
    return run_windows_host(m, w, padding, {"bnm_emulate_windows_topk", kEngineEmul, kInF32, true, nullptr, 0,
                                            {nullptr, nullptr, nullptr, {k, classes, scores}}, {}, nullptr, true});
}

// host buffers: n <= kSmallBatch images share a launch with concurrent small calls, larger batches run the chunked pipeline
extern "C" int bnm_infer_batch(bnm_model *m, const int8_t *images, size_t n, int32_t *logits, uint32_t *labels) {
    return run_call(m, {"bnm_infer_batch", kEngineC, kInI8, false, images, n, {logits, labels}, {}, nullptr, true});   // host buffers
}

// host buffers: the chunked pipeline of bnm_infer_batch, k classes (and k scores) per image copied back
extern "C" int bnm_infer_topk(bnm_model *m, const int8_t *images, size_t n, uint32_t k, uint32_t *classes, int32_t *scores) {
    return run_call(m, {"bnm_infer_topk", kEngineC, kInI8, true, images, n, {nullptr, nullptr, nullptr, {k, classes, scores}}, {}, nullptr,
                        true});   // host buffers
}

extern "C" int bnm_emulate_inference_quantized(bnm_model *m, const float *images, size_t n, double *logits) {
    return run_call(m, {"bnm_emulate_inference_quantized", kEngineEmul, kInF32, false, images, n, {logits}, {}, nullptr, true,
                        true});   // host buffers, logits required
}

// -----------------------------------------------------------------------------------------------
// reference-named symbols (BitNetMCU_inference.h:15-60): one item, abort on failure -- never a CPU path
// -----------------------------------------------------------------------------------------------
static void die(const char *fn) {
    fprintf(stderr, "bitnetmcu_b200: %s failed: %s\n", fn, g_err.c_str());
    abort();
}

extern "C" uint32_t ReLUNorm(int32_t *input, int8_t *output, uint32_t n_input) {
    uint32_t pos = 255;
    if (bnm_relunorm_batch(input, output, &pos, n_input, 1) != 0) die("ReLUNorm");
    return pos;
}
extern "C" void processfclayer(int8_t *activations, const uint32_t *weights, int32_t bits_per_weight, uint32_t n_input,
                               uint32_t n_output, int32_t *output) {
    if (bnm_processfclayer_batch(activations, weights, bits_per_weight, n_input, n_output, output, 1, 0) != 0) die("processfclayer");
}
extern "C" int32_t *processconv33ReLU(int32_t *activations, const int8_t *weights, uint32_t xy_input, uint32_t n_shift, int32_t *output) {
    if (bnm_conv33relu_batch(activations, weights, 1, xy_input, n_shift, output, 1) != 0) die("processconv33ReLU");
    return output + (size_t)(xy_input - 2) * (xy_input - 2);
}
extern "C" int32_t *processmaxpool22(int32_t *activations, uint32_t xy_input, int32_t *output) {
    if (bnm_maxpool22_batch(activations, xy_input, output, 1) != 0) die("processmaxpool22");
    return output + (size_t)(xy_input / 2) * (xy_input / 2);
}
