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

struct PipeSlot {
    cudaStream_t stream = nullptr;
    DevBuf<int8_t> d_images;
    DevBuf<int32_t> d_logits;
    DevBuf<uint32_t> d_labels;
    DevBuf<uint32_t> d_classes;   // bnm_infer_topk: the chunk's classes (its scores go to d_logits)
};

// One staging generation of the small-batch path (infer_small): the rows of every call that joined it, in arrival order.
struct SmallGen {
    PinnedBuf<int8_t> h_in;     // [kSmallBatch][img_bytes]
    PinnedBuf<int32_t> h_out;   // logits [rows][n_classes] when a member asks for them, then labels [rows]
    DevBuf<int8_t> d_in;        // their device counterparts
    DevBuf<int32_t> d_out;
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
    // every call's device scratch comes from this pool, stream-ordered on the call's stream (Scratch)
    cudaMemPool_t pool = nullptr;
    // host pipeline: the large host calls take turns on host_mu
    std::mutex host_mu;
    PipeSlot slots[3];
    // small-batch path of bnm_infer_batch (the reference's own calling pattern: one image per Inference() call,
    // test_inference.py:146-150): pinned staging buffers, one stream, one synchronisation per shared launch
    SmallBatcher small;
    bool verbose = false;           // BNM_VERBOSE at model creation: the top-k entries name their route on every call
    int small_zero_copy = 1;   // 0: H2D + D2H copies; 1 (default): the kernel writes results
                               // straight into mapped pinned host memory; 2: ... and reads the images from it (TMA over PCIe)
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

static void free_fc_layer(FcLayerDev &L) {
    cudaFree(L.dense_a);
    cudaFree(L.dense_b);
    cudaFree(L.quad_a);
    cudaFree(L.quad_b);
    L.dense_a = L.dense_b = nullptr;
    L.quad_a = L.quad_b = nullptr;
}

// one FC layer's packed weights (device, zero padded past the end) decoded into its int8 planes, the residual ones only where they
// are needed.  On failure nothing stays allocated.
static cudaError_t decode_fc_layer(const void *d_packed, int32_t enc, uint32_t n_in, uint32_t n_out, int nf4_ext, FcLayerDev &L) {
    L.enc = enc;
    L.n_in = n_in;
    L.n_out = n_out;
    L.k_pad = round_up(std::max(n_in, 1u), 32);
    L.n_pad = round_up(n_out, 16);
    const size_t plane = (size_t)L.k_pad * L.n_pad;
    DevBuf<int> d_flag;
    int flag = 0;
    cudaError_t e = cudaMalloc(&L.dense_a, plane);
    if (e == cudaSuccess) e = cudaMalloc(&L.dense_b, plane);
    if (e == cudaSuccess) e = cudaMalloc(&L.quad_a, plane);
    if (e == cudaSuccess) e = cudaMalloc(&L.quad_b, plane);
    if (e == cudaSuccess) e = d_flag.grow(sizeof(int), true);
    if (e == cudaSuccess) {
        launch_decode_fc(d_packed, enc, n_in, n_out, L.k_pad, L.n_pad, L.dense_a, L.dense_b, L.quad_a, L.quad_b, nf4_ext, d_flag.p, 0);
        e = cudaMemcpy(&flag, d_flag.p, sizeof(int), cudaMemcpyDeviceToHost);
    }
    if (e != cudaSuccess) {
        free_fc_layer(L);
    } else if (!flag) {   // no residual plane needed (everything but FP130 layers that contain +128)
        cudaFree(L.dense_b);
        cudaFree(L.quad_b);
        L.dense_b = nullptr;
        L.quad_b = nullptr;
    }
    return e;
}

static void free_fc_dev(bnm_model *m) {
    for (auto &L : m->fc) free_fc_layer(L);
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
        if (cudaError_t e = decode_fc_layer(H.d_packed, H.enc, H.n_in, H.n_out, m->nf4_ext, L)) {   // nothing half-built stays behind
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
    m->plan = fc_chain_plan_create(m->fc.data(), (int)m->fc.size(), in_bytes, m->device, m->sm_count, err, sizeof(err));
    m->plan_err = err;
    fc_chain_plan_set_overlap(m->plan, effective_overlap(m));
    return 0;
}

// One call's device scratch: stream-ordered allocations from the model's pool on the call's stream, handed back on that stream
// once the call has enqueued the work that uses them (the destructor).  Two calls in flight never share a byte of it, whatever
// their threads and streams, and no call waits on the host for another.  The pool keeps what it has (its release threshold
// is unbounded), so in steady state an allocation neither reaches the driver nor synchronises.
struct Scratch {
    cudaMemPool_t pool;
    cudaStream_t st;
    std::vector<void *> held;
    Scratch(const bnm_model *m, cudaStream_t s) : pool(m->pool), st(s) {}
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

// the kernels of the emulator (emulate_device): fc_emul_kernel on float images; fc_emul_i8_kernel after the scaling kernel (FC)
// or k_cnn_emul_frontend (CNN); or the emulation kernels layer by layer
enum EmulRoute { kEmulFloatRow, kEmulInt8Row, kEmulLayers };
static EmulRoute emul_route(const bnm_model *m) {
    const bool cnn = m->model_class == BNM_MODEL_CNNMNIST;
    if (bnm_model_active_path(m) != BNM_PATH_TCGEN05 || (cnn && m->channels > kCnnEmulMaxChannels)) return kEmulLayers;
    return !cnn && fc_chain_has_form(m->plan, kFormEmulFloat) ? kEmulFloatRow : kEmulInt8Row;
}
// the kernel that makes the emulator's int8 rows from float images on its row routes (emulate_device)
static const char *emul_rows_kernel(const bnm_model *m) {
    return m->model_class == BNM_MODEL_CNNMNIST ? "k_cnn_emul_frontend" : "k_quantize_images";
}

// bnm_compare_engines_device: fc_engines_kernel for the models both float-input rows serve, else the two entries' routes and
// k_engine_counts
static bool engines_fused(const bnm_model *m) {
    return bnm_model_active_path(m) == BNM_PATH_TCGEN05 && m->model_class == BNM_MODEL_FCMNIST && fc_chain_has_form(m->plan, kFormEngines);
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
    if (rc == 0) rc = build_fc_dev(m);
    if (rc == 0 && m->d_err.grow(sizeof(int), true) != cudaSuccess) rc = fail(BNM_E_CUDA, "cudaMalloc failed");
    if (rc == 0) {
        cudaMemPoolProps props = {};
        props.allocType = cudaMemAllocationTypePinned;
        props.location.type = cudaMemLocationTypeDevice;
        props.location.id = device;
        uint64_t keep = UINT64_MAX;   // never hand memory back to the device: steady-state calls neither allocate nor synchronise
        if (cudaMemPoolCreate(&m->pool, &props) != cudaSuccess || cudaMemPoolSetAttribute(m->pool, cudaMemPoolAttrReleaseThreshold, &keep) != cudaSuccess)
            rc = fail(BNM_E_CUDA, "scratch memory pool: %s", cudaGetErrorString(cudaGetLastError()));
    }
    if (rc == 0) {
        if (const char *e = getenv("BNM_CNN_FRONTEND")) m->cnn_frontend = std::max(0, std::min(2, atoi(e)));   // development override, read once per model
        if (const char *e = getenv("BNM_SMALL_ZC")) m->small_zero_copy = std::max(0, std::min(2, atoi(e)));     // development knob, likewise
        for (auto &s : m->slots)
            if (cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking) != cudaSuccess) { rc = fail(BNM_E_CUDA, "cudaStreamCreate failed"); break; }
        if (rc == 0 && cudaStreamCreateWithFlags(&m->small.stream, cudaStreamNonBlocking) != cudaSuccess) rc = fail(BNM_E_CUDA, "cudaStreamCreate failed");
    }
    if (rc != 0) { std::string keep = g_err; bnm_model_destroy(m); g_err = keep; return rc; }
    m->verbose = getenv("BNM_VERBOSE") != nullptr;
    if (m->verbose) {   // diagnostics: the kernels bnm_emulate_batch_device runs on the default path
        const EmulRoute r = emul_route(m);
        if (r == kEmulLayers) fprintf(stderr, "bitnetmcu_b200: emulator route: layer by layer\n");
        else if (r == kEmulFloatRow) fprintf(stderr, "bitnetmcu_b200: emulator route: %s\n", fc_chain_form_name(m->plan, kFormEmulFloat));
        else fprintf(stderr, "bitnetmcu_b200: emulator route: %s + %s\n", emul_rows_kernel(m), fc_chain_form_name(m->plan, kFormEmulInt8));
        // and the kernels of bnm_compare_engines_device
        if (engines_fused(m)) fprintf(stderr, "bitnetmcu_b200: engines route: %s\n", fc_chain_form_name(m->plan, kFormEngines));
        else fprintf(stderr, "bitnetmcu_b200: engines route: bnm_infer_batch_device_f32 + bnm_emulate_batch_device + k_engine_counts\n");
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
    if (m->pool) cudaMemPoolDestroy(m->pool);   // every call's scratch went back to it before the synchronisation above
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
static const size_t kLayeredChunk = 1 << 17;   // images per pass of the layer-by-layer path (bounds its scratch)
static const size_t kFusedCnnChunk = 1 << 20;  // fused path, CNN models: images per front-end + FC launch pair (256 B of features each)

// FC chain, one CUDA-core kernel per layer: input int8 [n][in_stride].  Without logits the last layer's accumulators go to the
// scratch (n x max_nout) like every other layer's, and only its ReLUNorm's argmax leaves it.
static int run_fc_layers(bnm_model *m, const int8_t *in, uint32_t in_stride, size_t n, int32_t *logits, uint32_t *labels,
                         const LayerScratch &ls, cudaStream_t st) {
    const int8_t *act = in;
    uint32_t stride = in_stride;
    const size_t nl = m->fc.size();
    for (size_t l = 0; l < nl; l++) {
        const bool last = l + 1 == nl;
        int32_t *acc = last && logits ? logits : ls.acc;
        if (!launch_fc_dp4a(act, stride, m->fc[l], acc, n, st))
            return fail(BNM_E_UNSUPPORTED, "FC layer %zu: %u inputs need more shared memory than an SM has (layer kernel stages 128 rows)", l, m->fc[l].n_in);
        if (last) {
            if (labels) launch_relunorm(acc, m->fc[l].n_out, nullptr, 0, labels, n, st);
        } else {
            int8_t *next = ls.act[l & 1];
            uint32_t next_stride = m->fc[l + 1].k_pad;
            launch_relunorm(acc, m->fc[l].n_out, next, next_stride, nullptr, n, st);
            act = next;
            stride = next_stride;
        }
    }
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

// images per chunk of the C engine on int8 images; 0: one launch whatever the batch (FC models on the fused path)
static size_t c_engine_chunk(const bnm_model *m, bool fused) {
    if (!fused) return kLayeredChunk;
    return m->model_class == BNM_MODEL_CNNMNIST ? kFusedCnnChunk : 0;
}

extern "C" int bnm_infer_launch_count(const bnm_model *m, size_t n) {
    if (!m || n == 0) return 0;
    const bool fused = bnm_model_active_path(m) == BNM_PATH_TCGEN05;
    const size_t chunk = c_engine_chunk(m, fused);
    if (!chunk) return 1;
    int per = m->model_class == BNM_MODEL_CNNMNIST ? 1 : 0;
    per += fused ? 1 : (int)(2 * m->fc.size());   // fc + relunorm per layer (last relunorm = labels)
    return (int)((n + chunk - 1) / chunk * per);
}

// a call must produce something: logits, labels or (gather) a destination in another buffer
static bool has_output(const int32_t *logits, const uint32_t *labels, const GatherDst *gather) {
    return logits || labels || (gather && (gather->n_labels_dst || gather->n_logits_dst));
}

// the top-k outputs of a call from image b on (T: the type of its scores)
template <class T> static TopKOutputs topk_from(const TopKOutputs &t, size_t b) {
    return TopKOutputs{t.k, t.classes ? t.classes + b * t.k : nullptr, t.scores ? static_cast<T *>(t.scores) + b * t.k : nullptr};
}

// The C engine on int8 images on st, arguments checked -> out: logits int32 [n][n_classes], labels and gather, or with topk.k > 0
// the k best classes of every image and their int32 scores.  FC models on the fused path in one launch, every other model in chunks
// (CNN front-end, then the fused launch, or the layer-by-layer chain and for top-k k_topk_rows on its int32 accumulators).
// The chunks' scratch (CNN features, the layer-by-layer path's buffers) is this call's own, for one chunk.
static int run_c_engine(bnm_model *m, const int8_t *images, size_t n, const FcOutputs &out, cudaStream_t st) {
    const bool fused = bnm_model_active_path(m) == BNM_PATH_TCGEN05;
    const bool cnn = m->model_class == BNM_MODEL_CNNMNIST;
    const uint32_t k = out.topk.k;
    const FcForm form = k ? kFormTopK : kFormInt8;
    const char *kernel = k ? "top-k" : "FC";
    const size_t chunk_max = c_engine_chunk(m, fused);
    if (!chunk_max) {
        int rc = fc_chain_launch(m->plan, form, images, n, out, st);
        return rc ? fail(BNM_E_CUDA, "fused %s kernel launch failed (%d): %s", kernel, rc, cudaGetErrorString(cudaGetLastError())) : 0;
    }
    const size_t chunk = std::min(n, chunk_max);
    Scratch scratch(m, st);
    LayerScratch ls;
    int8_t *feat = nullptr;
    if (!fused) CU_TRY(layer_scratch(m, scratch, chunk, ls));
    if (cnn) CU_TRY(scratch.get(&feat, chunk * m->feat_stride));
    int rc = 0;
    for (size_t b = 0; b < n; b += chunk) {
        const size_t nb = std::min(chunk, n - b);
        const int8_t *fc_in = images + b * m->img_bytes;
        uint32_t fc_stride = m->img_bytes;
        if (cnn) {
            if ((rc = run_cnn_front(m, fc_in, nb, feat, st))) return rc;
            fc_in = feat;
            fc_stride = m->feat_stride;
        }
        int32_t *lg = out.logits ? static_cast<int32_t *>(out.logits) + b * m->n_classes : nullptr;
        FcOutputs o{lg, out.labels ? out.labels + b : nullptr, nullptr, topk_from<int32_t>(out.topk, b)};
        if (fused) {
            GatherDst gchunk;
            if (out.gather) { gchunk = *out.gather; gchunk.row_offset += b; o.gather = &gchunk; }
            if ((rc = fc_chain_launch(m->plan, form, fc_in, nb, o, st)))
                return fail(BNM_E_CUDA, "fused %s kernel launch failed (%d)", kernel, rc);
        } else {
            if ((rc = run_fc_layers(m, fc_in, fc_stride, nb, lg, o.labels, ls, st))) return rc;
            if (k) launch_topk_rows(ls.acc, m->n_classes, k, o.topk.classes, static_cast<int32_t *>(o.topk.scores), nb, st);   // last layer's accumulators
        }
    }
    return launch_status();
}

static int infer_device_impl(bnm_model *m, const int8_t *images, size_t n, int32_t *logits, uint32_t *labels, const GatherDst *gather, void *stream) {
    if (!m || (n && !images)) return fail(BNM_E_ARG, "bnm_infer_batch_device: null argument");
    if (n && !has_output(logits, labels, gather)) return fail(BNM_E_ARG, "bnm_infer_batch_device: no output (logits, labels and gather destinations all absent)");
    if (n == 0) return 0;
    if ((uintptr_t)images & 15) return fail(BNM_E_ARG, "the device image buffer must be 16-byte aligned (TMA)");
    if (logits && ((uintptr_t)logits & 7)) return fail(BNM_E_ARG, "the device logits buffer must be 8-byte aligned (64-bit row stores)");
    CU_TRY(cudaSetDevice(m->device));
    if (gather && bnm_model_active_path(m) != BNM_PATH_TCGEN05)
        return fail(BNM_E_UNSUPPORTED, "the fused result exchange needs the fused tensor-core path (model: %s)", m->plan_err.c_str());
    return run_c_engine(m, images, n, FcOutputs{logits, labels, gather}, static_cast<cudaStream_t>(stream));
}

extern "C" int bnm_infer_batch_device(bnm_model *m, const int8_t *images, size_t n, int32_t *logits, uint32_t *labels, void *stream) {
    return infer_device_impl(m, images, n, logits, labels, nullptr, stream);
}

extern "C" int bnm_infer_batch_device_gather(bnm_model *m, const int8_t *images, size_t n, int32_t *logits, uint32_t *labels,
                                             const bnm_gather *gather, void *stream) {
    static_assert(sizeof(bnm_gather) == sizeof(GatherDst), "bnm_gather and GatherDst must share their layout");
    if (gather && (gather->n_labels_dst > BNM_MAX_GATHER_DST || gather->n_logits_dst > BNM_MAX_GATHER_DST))
        return fail(BNM_E_ARG, "at most %d gather destinations", BNM_MAX_GATHER_DST);
    if (gather)
        for (uint32_t d = 0; d < gather->n_logits_dst; d++)
            if ((uintptr_t)gather->logits_dst[d] & 7) return fail(BNM_E_ARG, "gather logits buffers must be 8-byte aligned");
    return infer_device_impl(m, images, n, logits, labels, reinterpret_cast<const GatherDst *>(gather), stream);
}

// -----------------------------------------------------------------------------------------------
// peer memory plumbing for the fused result exchange: cudaMalloc'd buffers exported / opened through CUDA IPC
// -----------------------------------------------------------------------------------------------
extern "C" int bnm_device_alloc(int device, size_t bytes, void **out) {
    if (!out) return fail(BNM_E_ARG, "bnm_device_alloc: null argument");
    *out = nullptr;
    if (int rc = require_device_index(device)) return rc;
    CU_TRY(cudaSetDevice(device));
    CU_TRY(cudaMalloc(out, bytes ? bytes : 16));
    return 0;
}
extern "C" void bnm_device_free(void *p) { if (p) cudaFree(p); }
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
    if (g[1].d_out.p) return 0;
    CU_TRY(cudaSetDevice(m->device));
    const size_t in_bytes = kSmallBatch * (size_t)m->img_bytes, out_bytes = kSmallBatch * ((size_t)m->n_classes + 1) * 4;
    cudaError_t e = cudaSuccess;
    for (int i = 0; i < 2 && e == cudaSuccess; i++) {
        e = g[i].h_in.grow(in_bytes);
        if (e == cudaSuccess) e = g[i].h_out.grow(out_bytes);
        if (e == cudaSuccess) e = g[i].d_in.grow(in_bytes);
        if (e == cudaSuccess) e = g[i].d_out.grow(out_bytes);
    }
    if (e == cudaSuccess) return 0;
    for (int i = 0; i < 2; i++) { g[i].h_in.release(); g[i].h_out.release(); g[i].d_in.release(); g[i].d_out.release(); }
    return fail(-100 - (int)e, "small-batch staging buffers: %s", cudaGetErrorString(e));
}

// One generation's rows through the GPU: one copy in, one launch, one copy out (or zero-copy), one synchronisation.
static int small_launch(bnm_model *m, SmallGen &g) {
    CU_TRY(cudaSetDevice(m->device));
    cudaStream_t st = m->small.stream;
    const size_t n = g.rows;
    const int8_t *d_in = g.d_in.p;
    int32_t *d_out = g.d_out.p;
    if (m->small_zero_copy >= 2) CU_TRY(cudaHostGetDevicePointer(reinterpret_cast<void **>(const_cast<int8_t **>(&d_in)), g.h_in.p, 0));
    else CU_TRY(cudaMemcpyAsync(g.d_in.p, g.h_in.p, n * (size_t)m->img_bytes, cudaMemcpyHostToDevice, st));
    if (m->small_zero_copy >= 1) CU_TRY(cudaHostGetDevicePointer(reinterpret_cast<void **>(&d_out), g.h_out.p, 0));
    const size_t n_log = g.logits ? n * (size_t)m->n_classes : 0;   // labels-only batches: the labels start the staging buffer
    uint32_t *d_lab = reinterpret_cast<uint32_t *>(d_out + n_log);
    int rc = bnm_infer_batch_device(m, d_in, n, g.logits ? d_out : nullptr, g.labels ? d_lab : nullptr, st);
    if (rc) return rc;
    if (m->small_zero_copy == 0) CU_TRY(cudaMemcpyAsync(g.h_out.p, g.d_out.p, (n_log + (g.labels ? n : 0)) * 4, cudaMemcpyDeviceToHost, st));
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
// that joins a generation must never wait on the runtime while the launch in flight is being synchronised.
static int infer_small(bnm_model *m, const int8_t *images, size_t n, int32_t *logits, uint32_t *labels) {
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

// the C engine on host buffers in chunks of chunk_images, each through one slot's buffers: images in, run_c_engine, out's arrays
// back.  Synchronous.
static int infer_pipelined(bnm_model *m, const int8_t *images, size_t n, const FcOutputs &out) {
    std::lock_guard<std::mutex> turn(m->host_mu);   // large host calls take turns: each one keeps the copy engines busy alone
    const size_t chunk = std::min(n, m->chunk_images), k = out.topk.k;
    // per image, in 4-byte words: d_logits holds the logits or the top-k scores (bnm_infer_batch sizes it and d_labels whether or
    // not it takes them), d_classes the top-k classes
    const size_t n_logits = k ? (out.topk.scores ? k : 0) : m->n_classes, n_labels = k ? 0 : 1;
    bool small = false;
    for (auto &s : m->slots)
        small = small || s.d_images.bytes < chunk * m->img_bytes || s.d_classes.bytes < chunk * k * 4 ||
                s.d_logits.bytes < chunk * n_logits * 4 || s.d_labels.bytes < chunk * n_labels * 4;
    if (small) {
        for (auto &s : m->slots) CU_TRY(cudaStreamSynchronize(s.stream));   // no chunk of an earlier call may still use a buffer that is reallocated
        for (auto &s : m->slots) {
            CU_TRY(s.d_images.grow(chunk * (size_t)m->img_bytes));
            CU_TRY(s.d_classes.grow(chunk * k * 4));
            CU_TRY(s.d_logits.grow(chunk * n_logits * 4));
            CU_TRY(s.d_labels.grow(chunk * n_labels * 4));
        }
    }
    // every chunk's scratch is its own (run_c_engine): the chunks of every path overlap in time on all three streams
    int32_t *h_logits = static_cast<int32_t *>(k ? out.topk.scores : out.logits);   // where d_logits goes
    size_t c = 0;
    for (size_t b = 0; b < n; b += chunk, c++) {
        const size_t nb = std::min(chunk, n - b);
        PipeSlot &s = m->slots[c % 3];
        CU_TRY(cudaMemcpyAsync(s.d_images.p, images + b * m->img_bytes, nb * (size_t)m->img_bytes, cudaMemcpyHostToDevice, s.stream));
        const FcOutputs d{out.logits ? s.d_logits.p : nullptr, out.labels ? s.d_labels.p : nullptr, nullptr,
                         {(uint32_t)k, s.d_classes.p, out.topk.scores ? s.d_logits.p : nullptr}};
        if (int rc = run_c_engine(m, s.d_images.p, nb, d, s.stream)) return rc;
        if (k) CU_TRY(cudaMemcpyAsync(out.topk.classes + b * k, s.d_classes.p, nb * k * 4, cudaMemcpyDeviceToHost, s.stream));
        if (h_logits) CU_TRY(cudaMemcpyAsync(h_logits + b * n_logits, s.d_logits.p, nb * n_logits * 4, cudaMemcpyDeviceToHost, s.stream));
        if (out.labels) CU_TRY(cudaMemcpyAsync(out.labels + b, s.d_labels.p, nb * 4, cudaMemcpyDeviceToHost, s.stream));
    }
    for (auto &s : m->slots) CU_TRY(cudaStreamSynchronize(s.stream));
    return 0;
}

extern "C" int bnm_infer_batch(bnm_model *m, const int8_t *images, size_t n, int32_t *logits, uint32_t *labels) {
    if (!m || (n && !images)) return fail(BNM_E_ARG, "bnm_infer_batch: null argument");
    if (n && !logits && !labels) return fail(BNM_E_ARG, "bnm_infer_batch: no output (logits and labels both NULL)");
    if (n == 0) return 0;
    if (n <= kSmallBatch && n <= m->chunk_images) return infer_small(m, images, n, logits, labels);   // sets the device where it launches
    CU_TRY(cudaSetDevice(m->device));
    return infer_pipelined(m, images, n, FcOutputs{logits, labels});
}

extern "C" void *bnm_host_alloc(size_t bytes) {
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); fail(BNM_E_CUDA, "cudaHostAlloc(%zu) failed", bytes); return nullptr; }
    return p;
}
extern "C" void bnm_host_free(void *p) { if (p) cudaFreeHost(p); }

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

extern "C" int bnm_processfclayer_batch(const int8_t *activations, const uint32_t *weights, int32_t enc, uint32_t n_input,
                                        uint32_t n_output, int32_t *output, size_t n, int nf4_extension) {
    if (int rc = require_device()) return rc;
    if (n == 0 || n_output == 0) return 0;
    if (!activations || !weights || !output) return fail(BNM_E_ARG, "bnm_processfclayer_batch: null argument");
    const size_t need = packed_weight_bytes(enc, n_input, n_output);
    DevBuf<uint8_t> packed;
    if (packed.grow(need + 16)) return fail(BNM_E_CUDA, "cudaMalloc failed");
    CU_TRY(cudaMemset(packed.p, 0, need + 16));
    if (need) CU_TRY(cudaMemcpy(packed.p, weights, need, cudaMemcpyHostToDevice));
    FcLayerDev L;
    if (cudaError_t e = decode_fc_layer(packed.p, enc, n_input, n_output, nf4_extension, L))
        return fail(BNM_E_CUDA, "weight decode of an FC layer failed: %s", cudaGetErrorString(e));
    struct Planes { FcLayerDev &L; ~Planes() { free_fc_layer(L); } } planes{L};   // L's planes are freed on every return below
    DevBuf<int8_t> act;
    DevBuf<int32_t> out;
    if (act.grow(n * (size_t)L.k_pad) || out.grow(n * (size_t)n_output * 4)) return fail(BNM_E_CUDA, "cudaMalloc failed");
    CU_TRY(cudaMemset(act.p, 0, n * (size_t)L.k_pad));
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
    if (valid_in) CU_TRY(cudaMemcpy2D(act.p, L.k_pad, activations, n_input, valid_in, n, cudaMemcpyHostToDevice));
    if (!launch_fc_dp4a(act.p, L.k_pad, L, out.p, n, 0))
        return fail(BNM_E_UNSUPPORTED, "processfclayer: n_input %u needs more shared memory than an SM has (layer kernel stages 128 rows)", n_input);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpy(output, out.p, n * (size_t)n_output * 4, cudaMemcpyDeviceToHost));
    return 0;
}

extern "C" int bnm_relunorm_batch(const int32_t *input, int8_t *output, uint32_t *argmax, uint32_t n_input, size_t n) {
    if (int rc = require_device()) return rc;
    if (n == 0) return 0;
    if (n_input == 0) {   // inference.c:24-37: nothing is scanned, position stays 255
        if (argmax) for (size_t i = 0; i < n; i++) argmax[i] = 255;
        return 0;
    }
    if (!input) return fail(BNM_E_ARG, "bnm_relunorm_batch: null input");
    DevBuf<int32_t> in;
    DevBuf<int8_t> out;
    DevBuf<uint32_t> am;
    if (in.grow(n * (size_t)n_input * 4) || out.grow(n * (size_t)n_input) || am.grow(n * 4)) return fail(BNM_E_CUDA, "cudaMalloc failed");
    CU_TRY(cudaMemcpy(in.p, input, n * (size_t)n_input * 4, cudaMemcpyHostToDevice));   // copied first: output may alias input
    launch_relunorm(in.p, n_input, output ? out.p : nullptr, n_input, am.p, n, 0);
    CU_TRY(cudaGetLastError());
    if (argmax) CU_TRY(cudaMemcpy(argmax, am.p, n * 4, cudaMemcpyDeviceToHost));
    else CU_TRY(cudaDeviceSynchronize());
    if (output) CU_TRY(cudaMemcpy(output, out.p, n * (size_t)n_input, cudaMemcpyDeviceToHost));
    return 0;
}

extern "C" int bnm_conv33relu_batch(const int32_t *activations, const int8_t *weights, uint32_t n_w, uint32_t xy, uint32_t n_shift,
                                    int32_t *output, size_t n) {
    if (int rc = require_device()) return rc;
    if (n == 0 || xy < 3) return 0;
    if (!activations || !weights || !output || n_w == 0) return fail(BNM_E_ARG, "bnm_conv33relu_batch: null argument");
    const size_t in_el = n * (size_t)xy * xy, out_el = n * (size_t)(xy - 2) * (xy - 2);
    DevBuf<int32_t> in, out;
    DevBuf<int8_t> w;
    if (in.grow(in_el * 4) || w.grow((size_t)n_w * 9) || out.grow(out_el * 4)) return fail(BNM_E_CUDA, "cudaMalloc failed");
    CU_TRY(cudaMemcpy(in.p, activations, in_el * 4, cudaMemcpyHostToDevice));
    CU_TRY(cudaMemcpy(w.p, weights, (size_t)n_w * 9, cudaMemcpyHostToDevice));
    launch_conv33relu(in.p, w.p, n_w, xy, n_shift, out.p, n, 0);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpy(output, out.p, out_el * 4, cudaMemcpyDeviceToHost));
    return 0;
}

extern "C" int bnm_maxpool22_batch(const int32_t *activations, uint32_t xy, int32_t *output, size_t n) {
    if (int rc = require_device()) return rc;
    if (n == 0 || xy < 2) return 0;
    if (!activations || !output) return fail(BNM_E_ARG, "bnm_maxpool22_batch: null argument");
    const size_t in_el = n * (size_t)xy * xy, out_el = n * (size_t)(xy / 2) * (xy / 2);
    DevBuf<int32_t> in, out;
    if (in.grow(in_el * 4) || out.grow(out_el * 4)) return fail(BNM_E_CUDA, "cudaMalloc failed");
    CU_TRY(cudaMemcpy(in.p, activations, in_el * 4, cudaMemcpyHostToDevice));
    launch_maxpool22(in.p, xy, out.p, n, 0);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpy(output, out.p, out_el * 4, cudaMemcpyDeviceToHost));
    return 0;
}

extern "C" int bnm_quantize_images_device(const float *images, size_t n, uint32_t elems, int8_t *out, void *stream) {
    if (int rc = require_device()) return rc;
    if (n == 0 || elems == 0) return 0;
    if (!images || !out) return fail(BNM_E_ARG, "bnm_quantize_images_device: null argument");
    launch_quantize_images(images, elems, out, n, static_cast<cudaStream_t>(stream));
    return launch_status();
}

// float images -> logits / labels on the device.  FC models on the fused path (rows of <= 256 elements, <= 16 classes): ONE kernel, the
// input scaling fused into its load stage.  Everything else: the scaling kernel into a scratch buffer, then the ordinary path.
extern "C" int bnm_infer_batch_device_f32(bnm_model *m, const float *images, size_t n, int32_t *logits, uint32_t *labels, void *stream) {
    if (!m || (n && !images)) return fail(BNM_E_ARG, "bnm_infer_batch_device_f32: null argument");
    if (n && !logits && !labels) return fail(BNM_E_ARG, "bnm_infer_batch_device_f32: no output (logits and labels both NULL)");
    if (n == 0) return 0;
    if ((uintptr_t)images & 15) return fail(BNM_E_ARG, "the device image buffer must be 16-byte aligned");
    if (logits && ((uintptr_t)logits & 7)) return fail(BNM_E_ARG, "the device logits buffer must be 8-byte aligned (64-bit row stores)");
    CU_TRY(cudaSetDevice(m->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool fused_fc = bnm_model_active_path(m) == BNM_PATH_TCGEN05 && m->model_class == BNM_MODEL_FCMNIST;
    if (fused_fc && fc_chain_has_form(m->plan, kFormFloat)) {
        int rc = fc_chain_launch(m->plan, kFormFloat, images, n, FcOutputs{logits, labels}, st);
        return rc ? fail(BNM_E_CUDA, "fused float-input kernel launch failed (%d): %s", rc, cudaGetErrorString(cudaGetLastError())) : 0;
    }
    Scratch scratch(m, st);
    int8_t *q;
    CU_TRY(scratch.get(&q, n * (size_t)m->img_bytes));
    launch_quantize_images(images, m->img_bytes, q, n, st);
    return bnm_infer_batch_device(m, q, n, logits, labels, stream);
}

extern "C" int bnm_quantize_images(const float *images, size_t n, uint32_t elems, int8_t *out) {
    if (int rc = require_device()) return rc;
    if (n == 0 || elems == 0) return 0;
    if (!images || !out) return fail(BNM_E_ARG, "bnm_quantize_images: null argument");
    DevBuf<float> in;
    DevBuf<int8_t> q;
    if (in.grow(n * (size_t)elems * 4) || q.grow(n * (size_t)elems)) return fail(BNM_E_CUDA, "cudaMalloc failed");
    CU_TRY(cudaMemcpy(in.p, images, n * (size_t)elems * 4, cudaMemcpyHostToDevice));
    launch_quantize_images(in.p, elems, q.p, n, 0);
    CU_TRY(cudaGetLastError());
    CU_TRY(cudaMemcpy(out, q.p, n * (size_t)elems, cudaMemcpyDeviceToHost));
    return 0;
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
//   * CNN models up to kCnnEmulMaxChannels channels: the front-end kernel k_cnn_emul_frontend, then fc_emul_i8_kernel on its features.
// BNM_PATH_LAYERS, models without a fused plan and wider CNN models run the emulation kernels layer by layer.
// -----------------------------------------------------------------------------------------------
int bnm::level_shift_of(int32_t enc) { return (enc == BNM_ENC_2BITSYM || enc == BNM_ENC_4BITSYM) ? 1 : 0; }
static const size_t kEmulChunkFc = 65536, kEmulChunkCnn = 2048;   // images per pass of the layer kernels (CNN: 2 x C kB of planes each)

// The emulator on device buffers, asynchronous on st: images float32 [n][img_bytes] -> logits float64 [n][n_classes] and / or labels
// (first maximum); or, with topk.k > 0, instead of both the k best classes of every image and their float64 scores (may be null).
// The routes other than fc_emul_kernel run in chunks through scratch of their own, for one chunk.
static int emulate_device(bnm_model *m, const float *images, size_t n, double *logits, uint32_t *labels, cudaStream_t st,
                          const TopKOutputs &topk = {}) {
    const size_t nl = m->fc.size();
    const bool cnn = m->model_class == BNM_MODEL_CNNMNIST;
    const uint32_t C = m->channels, elems = m->img_bytes, k = topk.k;
    const EmulRoute route = emul_route(m);
    if (route == kEmulFloatRow && !k) {   // fc_emul_kernel has no top-k form: top-k takes the int8 rows
        int rc = fc_chain_launch(m->plan, kFormEmulFloat, images, n, FcOutputs{logits, labels}, st);
        return rc ? fail(BNM_E_CUDA, "fused emulator kernel launch failed (%d): %s", rc, cudaGetErrorString(cudaGetLastError())) : 0;
    }
    if (route != kEmulLayers) {
        const size_t chunk = std::min(n, kFusedCnnChunk);
        Scratch scratch(m, st);
        int8_t *rows;   // the int8 emulator row's input: scaled images (FC) or front-end features (CNN)
        CU_TRY(scratch.get(&rows, chunk * (cnn ? m->feat_stride : elems)));
        for (size_t b = 0; b < n; b += chunk) {
            const size_t nb = std::min(chunk, n - b);
            if (!cnn) launch_quantize_images(images + b * elems, elems, rows, nb, st);   // BitNetMCU.py:435-436
            else if (!launch_cnn_emul_frontend(images + b * elems, m->d_conv[0].p, m->d_conv[1].p, m->d_conv[2].p, C, rows, m->feat_stride, nb, st))
                return fail(BNM_E_CUDA, "emulator CNN front-end: cannot opt in to its dynamic shared memory");
            const FcOutputs out{logits ? logits + b * m->n_classes : nullptr, labels ? labels + b : nullptr, nullptr, topk_from<double>(topk, b)};
            int rc = fc_chain_launch(m->plan, k ? kFormEmulTopK : kFormEmulInt8, rows, nb, out, st);
            if (rc) return fail(BNM_E_CUDA, "fused %s kernel launch failed (%d): %s", k ? "emulator top-k" : "int8 emulator", rc,
                                cudaGetErrorString(cudaGetLastError()));
        }
        return launch_status();
    }
    const size_t chunk = std::min(n, cnn ? kEmulChunkCnn : kEmulChunkFc);
    Scratch scratch(m, st);
    LayerScratch ls;   // accumulators and the two int8 activation buffers
    double *topk_logits;   // top-k: the logits of a chunk
    int8_t *q;             // the quantised images
    int32_t *planes[2];    // CNN models: int32 conv planes
    CU_TRY(layer_scratch(m, scratch, chunk, ls));
    CU_TRY(scratch.get(&topk_logits, k ? chunk * m->n_classes : 0));
    CU_TRY(scratch.get(&q, chunk * elems));
    for (auto &p : planes) CU_TRY(scratch.get(&p, cnn ? chunk * C * 256 : 0));
    int8_t *a0 = ls.act[0], *a1 = ls.act[1];
    for (size_t b = 0; b < n; b += chunk) {
        const size_t nb = std::min(chunk, n - b);
        launch_quantize_images(images + b * elems, elems, q, nb, st);   // BitNetMCU.py:435-436
        const int8_t *act = q;
        uint32_t stride = elems;
        if (cnn) {
            // conv (ReLU, no shift) -> per-image renormalisation, pools in between (BitNetMCU.py:459-526), planes [(image, channel)][xy*xy]
            int32_t *p0 = planes[0], *p1 = planes[1];
            launch_expand_image(q, p0, C, 256, nb, st);
            launch_conv33relu(p0, m->d_conv[0].p, C, 16, 0, p1, nb * C, st);
            launch_conv_renorm(p1, C * 196, nb, st);
            launch_conv33relu(p1, m->d_conv[1].p, C, 14, 0, p0, nb * C, st);
            launch_conv_renorm(p0, C * 144, nb, st);
            launch_maxpool22(p0, 12, p1, nb * C, st);
            launch_conv33relu(p1, m->d_conv[2].p, C, 6, 0, p0, nb * C, st);
            launch_conv_renorm(p0, C * 16, nb, st);
            launch_maxpool22(p0, 4, p1, nb * C, st);
            launch_i32_to_i8(p1, C * 4, a1, m->feat_stride, nb, st);   // flatten (C, 2, 2) -> features (BitNetMCU.py:443-445)
            act = a1;
            stride = m->feat_stride;
        }
        for (size_t l = 0; l < nl; l++) {
            if (!launch_fc_dp4a(act, stride, m->fc[l], ls.acc, nb, st)) return fail(BNM_E_UNSUPPORTED, "FC layer %zu too wide for the layer kernel", l);
            if (l + 1 == nl) break;   // no renormalisation for the last layer (BitNetMCU.py:528-530)
            int8_t *next = (l & 1) ? a1 : a0;   // CNN features sit in a1 and are dead once layer 0 has run
            const uint32_t next_stride = m->fc[l + 1].k_pad;
            launch_relunorm_emul(ls.acc, m->fc[l].n_out, level_shift_of(m->fc[l].enc), next, next_stride, nb, st);
            act = next;
            stride = next_stride;
        }
        double *lg = k ? topk_logits : logits ? logits + b * m->n_classes : nullptr;
        launch_emul_logits(ls.acc, m->n_classes, level_shift_of(m->fc[nl - 1].enc), lg, labels ? labels + b : nullptr, nb, st);
        if (k) {
            const TopKOutputs tk = topk_from<double>(topk, b);
            launch_topk_rows(lg, m->n_classes, k, tk.classes, static_cast<double *>(tk.scores), nb, st);
        }
    }
    return launch_status();
}

extern "C" int bnm_emulate_batch_device(bnm_model *m, const float *images, size_t n, double *logits, uint32_t *labels, void *stream) {
    if (!m || (n && !images)) return fail(BNM_E_ARG, "bnm_emulate_batch_device: null argument");
    if (n && !logits && !labels) return fail(BNM_E_ARG, "bnm_emulate_batch_device: no output (logits and labels both NULL)");
    if (n == 0) return 0;
    if ((uintptr_t)images & 15) return fail(BNM_E_ARG, "the device image buffer must be 16-byte aligned");
    if (logits && ((uintptr_t)logits & 7)) return fail(BNM_E_ARG, "the device logits buffer must be 8-byte aligned");
    CU_TRY(cudaSetDevice(m->device));
    return emulate_device(m, images, n, logits, labels, static_cast<cudaStream_t>(stream));
}

// host buffers: per chunk, images in -> emulate_device -> logits out, synchronously
extern "C" int bnm_emulate_inference_quantized(bnm_model *m, const float *images, size_t n, double *logits) {
    if (!m || (n && (!images || !logits))) return fail(BNM_E_ARG, "bnm_emulate_inference_quantized: null argument");
    if (n == 0) return 0;
    CU_TRY(cudaSetDevice(m->device));
    std::lock_guard<std::mutex> turn(m->host_mu);   // takes turns with the other large host calls, on the pipeline's first stream
    const size_t elems = m->img_bytes, ncls = m->n_classes;
    const size_t chunk = std::min(n, m->model_class == BNM_MODEL_CNNMNIST ? kEmulChunkCnn : kEmulChunkFc);
    cudaStream_t st = m->slots[0].stream;
    Scratch scratch(m, st);
    float *d_in;      // the device copies of a chunk's images and logits
    double *d_out;
    CU_TRY(scratch.get(&d_in, chunk * elems));
    CU_TRY(scratch.get(&d_out, chunk * ncls));
    for (size_t b = 0; b < n; b += chunk) {
        const size_t nb = std::min(chunk, n - b);
        CU_TRY(cudaMemcpyAsync(d_in, images + b * elems, nb * elems * sizeof(float), cudaMemcpyHostToDevice, st));
        if (int rc = emulate_device(m, d_in, nb, d_out, nullptr, st)) return rc;
        CU_TRY(cudaMemcpyAsync(logits + b * ncls, d_out, nb * ncls * sizeof(double), cudaMemcpyDeviceToHost, st));
        CU_TRY(cudaStreamSynchronize(st));
    }
    return 0;
}

// -----------------------------------------------------------------------------------------------
// Both engines in one call (test_inference.py:130-175): the C engine's and the emulator's labels of the same float images, and
// counts of their agreement and of their accuracy against truth.  The one-pass kernel where both float-input rows exist; every
// other model runs bnm_infer_batch_device_f32's and emulate_device's routes per chunk, into the caller's label buffers or the
// call's scratch, then k_engine_counts.
// -----------------------------------------------------------------------------------------------
static const size_t kEnginesChunk = 1 << 20;   // images per pass of the two routes (bounds the label scratch)

extern "C" int bnm_compare_engines_device(bnm_model *m, const float *images, size_t n, const uint32_t *truth, uint32_t *labels_c,
                                          uint32_t *labels_py, bnm_engine_counts *counts, void *stream) {
    static_assert(sizeof(bnm_engine_counts) == 4 * sizeof(unsigned long long), "bnm_engine_counts: four 64-bit counters");
    if (!m || (n && !images)) return fail(BNM_E_ARG, "bnm_compare_engines_device: null argument");
    if (!labels_c && !labels_py && !counts) return fail(BNM_E_ARG, "bnm_compare_engines_device: no output (labels_c, labels_py and counts all NULL)");
    if (truth && !counts) return fail(BNM_E_ARG, "bnm_compare_engines_device: truth without counts");
    if (n == 0) return 0;
    if ((uintptr_t)images & 15) return fail(BNM_E_ARG, "the device image buffer must be 16-byte aligned");
    if ((uintptr_t)counts & 7) return fail(BNM_E_ARG, "the device counts must be 8-byte aligned");
    CU_TRY(cudaSetDevice(m->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    auto *cnt = reinterpret_cast<unsigned long long *>(counts);
    if (engines_fused(m)) {
        int rc = fc_chain_launch(m->plan, kFormEngines, images, n, FcOutputs{nullptr, labels_c, nullptr, {}, {labels_py, truth, cnt}}, st);
        return rc ? fail(BNM_E_CUDA, "fused two-engine kernel launch failed (%d): %s", rc, cudaGetErrorString(cudaGetLastError())) : 0;
    }
    const size_t chunk = std::min(n, kEnginesChunk), elems = m->img_bytes;
    Scratch scratch(m, st);
    uint32_t *own[2];   // C / emulator labels the caller does not take
    CU_TRY(scratch.get(&own[0], counts && !labels_c ? chunk : 0));
    CU_TRY(scratch.get(&own[1], counts && !labels_py ? chunk : 0));
    for (size_t b = 0; b < n; b += chunk) {
        const size_t nb = std::min(chunk, n - b);
        const float *img = images + b * elems;
        uint32_t *lc = labels_c ? labels_c + b : own[0];
        uint32_t *lp = labels_py ? labels_py + b : own[1];
        if (lc)
            if (int rc = bnm_infer_batch_device_f32(m, img, nb, nullptr, lc, st)) return rc;
        if (lp)
            if (int rc = emulate_device(m, img, nb, nullptr, lp, st)) return rc;
        if (counts) launch_engine_counts(lc, lp, truth ? truth + b : nullptr, nb, m->n_classes, cnt, st);
    }
    return launch_status();
}

// -----------------------------------------------------------------------------------------------
// Top-k (section 8): the k best classes of every image and their scores -- the classes ranked by logit, highest first, ties to the
// lower class, so rank 0 is the label of the matching entry -- and no logits written anywhere.
//   * FC models on the fused path: one launch of fc_topk_kernel, whose epilogue ranks the classes in registers;
//   * CNN models on the fused path: the front-end into the feature scratch, then that kernel, in chunks of 2^20 images;
//   * BNM_PATH_LAYERS and models without a fused plan: the layer-by-layer chain into its int32 scratch (the emulator: its float64
//     logits into a chunk of scratch), then k_topk_rows.
// The float entry scales the images into its own scratch first; the emulator runs its own front-end (scaling kernel or CNN
// front-end) into its scratch, then fc_topk_kernel with its rule.
// -----------------------------------------------------------------------------------------------
static int topk_check(const bnm_model *m, const char *fn, const void *images, size_t n, uint32_t k, const uint32_t *classes,
                      const void *scores, uintptr_t score_align, uintptr_t image_align) {
    if (!m || (n && (!images || !classes))) return fail(BNM_E_ARG, "%s: null argument", fn);
    if (k < 1 || k > std::min<uint32_t>(m->n_classes, BNM_MAX_TOPK))
        return fail(BNM_E_ARG, "%s: k = %u, must be 1 .. min(n_classes = %u, %d)", fn, k, m->n_classes, BNM_MAX_TOPK);
    if ((uintptr_t)images & (image_align - 1)) return fail(BNM_E_ARG, "%s: the device image buffer must be %zu-byte aligned", fn, (size_t)image_align);
    if ((uintptr_t)classes & 3) return fail(BNM_E_ARG, "%s: the classes buffer must be 4-byte aligned", fn);
    if ((uintptr_t)scores & (score_align - 1)) return fail(BNM_E_ARG, "%s: the scores buffer must be %zu-byte aligned", fn, (size_t)score_align);
    return 0;
}

// the kernels of the C engine's top-k on int8 images, for the route line
static std::string topk_c_route(const bnm_model *m) {
    std::string s;
    if (m->model_class == BNM_MODEL_CNNMNIST)
        s = cnn_frontend_kernel(m->channels, m->xy0, m->cnn_frontend) == kCnnFrontendTensorCores ? "k_cnn_frontend16_tc + " : "k_cnn_frontend16 + ";
    if (bnm_model_active_path(m) == BNM_PATH_TCGEN05) return s + fc_chain_form_name(m->plan, kFormTopK);
    return s + "layer by layer + k_topk_rows<int32>";
}

extern "C" int bnm_infer_topk_device(bnm_model *m, const int8_t *images, size_t n, uint32_t k, uint32_t *classes, int32_t *scores, void *stream) {
    if (int rc = topk_check(m, "bnm_infer_topk_device", images, n, k, classes, scores, 4, 16)) return rc;
    if (n == 0) return 0;
    CU_TRY(cudaSetDevice(m->device));
    if (m->verbose) fprintf(stderr, "bitnetmcu_b200: topk route: bnm_infer_topk_device: %s\n", topk_c_route(m).c_str());
    return run_c_engine(m, images, n, FcOutputs{nullptr, nullptr, nullptr, {k, classes, scores}}, static_cast<cudaStream_t>(stream));
}

extern "C" int bnm_infer_topk_device_f32(bnm_model *m, const float *images, size_t n, uint32_t k, uint32_t *classes, int32_t *scores, void *stream) {
    if (int rc = topk_check(m, "bnm_infer_topk_device_f32", images, n, k, classes, scores, 4, 16)) return rc;
    if (n == 0) return 0;
    CU_TRY(cudaSetDevice(m->device));
    if (m->verbose) fprintf(stderr, "bitnetmcu_b200: topk route: bnm_infer_topk_device_f32: k_quantize_images + %s\n", topk_c_route(m).c_str());
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t chunk = std::min(n, kFusedCnnChunk), elems = m->img_bytes;
    Scratch scratch(m, st);
    int8_t *q;
    CU_TRY(scratch.get(&q, chunk * elems));
    for (size_t b = 0; b < n; b += chunk) {
        const size_t nb = std::min(chunk, n - b);
        launch_quantize_images(images + b * elems, (uint32_t)elems, q, nb, st);
        const FcOutputs out{nullptr, nullptr, nullptr, {k, classes + b * k, scores ? scores + b * k : nullptr}};
        if (int rc = run_c_engine(m, q, nb, out, st)) return rc;
    }
    return 0;
}

extern "C" int bnm_emulate_topk_device(bnm_model *m, const float *images, size_t n, uint32_t k, uint32_t *classes, double *scores, void *stream) {
    if (int rc = topk_check(m, "bnm_emulate_topk_device", images, n, k, classes, scores, 8, 16)) return rc;
    if (n == 0) return 0;
    CU_TRY(cudaSetDevice(m->device));
    if (m->verbose && emul_route(m) == kEmulLayers) fprintf(stderr, "bitnetmcu_b200: topk route: bnm_emulate_topk_device: layer by layer + k_topk_rows<double>\n");
    else if (m->verbose) fprintf(stderr, "bitnetmcu_b200: topk route: bnm_emulate_topk_device: %s + %s\n", emul_rows_kernel(m), fc_chain_form_name(m->plan, kFormEmulTopK));
    return emulate_device(m, images, n, nullptr, nullptr, static_cast<cudaStream_t>(stream), TopKOutputs{k, classes, scores});
}

// host buffers: the chunked pipeline of bnm_infer_batch, k classes (and k scores) per image copied back
extern "C" int bnm_infer_topk(bnm_model *m, const int8_t *images, size_t n, uint32_t k, uint32_t *classes, int32_t *scores) {
    if (int rc = topk_check(m, "bnm_infer_topk", images, n, k, classes, scores, 1, 1)) return rc;
    if (n == 0) return 0;
    CU_TRY(cudaSetDevice(m->device));
    if (m->verbose) fprintf(stderr, "bitnetmcu_b200: topk route: bnm_infer_topk: %s\n", topk_c_route(m).c_str());
    return infer_pipelined(m, images, n, FcOutputs{nullptr, nullptr, nullptr, {k, classes, scores}});
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
