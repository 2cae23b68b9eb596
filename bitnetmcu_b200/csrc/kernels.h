// kernels.h -- internal launch interface between the C-ABI layer (capi.cu) and the CUDA kernels.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace bnm {

constexpr int kMaxFcLayers = 8;
constexpr int kTileM = 128;  // images per MMA tile / per CTA tile of the layer kernels
constexpr int kMaxGatherDst = 8;   // destination buffers of the fused result exchange (one box: 8 GPUs)

// destinations of the fused result exchange: layout of bnm_gather (include/bitnetmcu_b200.h)
struct GatherDst {
    uint32_t n_labels_dst, n_logits_dst;
    uint32_t *labels_dst[kMaxGatherDst];
    int32_t *logits_dst[kMaxGatherDst];
    size_t row_offset;
    uint32_t labels_u8, reserved;
};

// One fully connected layer, decoded once at model build into dense int8 planes (K3 "weight pre-decode").
struct FcLayerDev {
    int32_t enc = 0;
    uint32_t n_in = 0, n_out = 0;   // as in the model header (Lk_incoming_weights / Lk_outgoing_weights)
    uint32_t k_pad = 0;             // n_in rounded up to 32 (one wgmma s8 K-step), zero padded
    uint32_t n_pad = 0;             // n_out rounded up to 16 (wgmma N granularity), zero padded
    int8_t *dense_a = nullptr;      // [n_pad][k_pad] row-major int8: clamp(w, -128, 127)
    int8_t *dense_b = nullptr;      // [n_pad][k_pad] residual plane w - clamp(w) (only FP130's +128), or null
    int4 *quad_a = nullptr;         // dp4a layout [(n_pad/4)][k_pad/4] of int4 = 4 outputs x 4 k (layer kernels)
    int4 *quad_b = nullptr;
};

// Lets `kernel` launch with `bytes` of dynamic shared memory on the current device: raises its
// cudaFuncAttributeMaxDynamicSharedMemorySize there when it is lower, never lowers it.  false (no error left pending) on failure.
bool raise_smem_limit(const void *kernel, size_t bytes);

// ---- weight decode (packed exportquant words -> dense planes); returns whether plane B is needed via *d_flag
void launch_decode_fc(const void *d_packed, int32_t enc, uint32_t n_in, uint32_t n_out, uint32_t k_pad, uint32_t n_pad,
                      int8_t *dense_a, int8_t *dense_b, int4 *quad_a, int4 *quad_b, int nf4_extension, int *d_flag,
                      cudaStream_t st);

// ---- layer-by-layer CUDA-core path (any shape)
// act int8 [n][act_stride] -> out int32 [n][n_out]; any stride and any byte alignment (rows that are not 4-byte aligned stage
// byte by byte), bytes of a row past act_stride read as zero
// false: the layer needs more shared memory than an SM has (k_pad > 1792: 128 staged rows of k_pad + 4 bytes in 227 kB)
bool launch_fc_dp4a(const int8_t *act, uint32_t act_stride, const FcLayerDev &L, int32_t *out, size_t n, cudaStream_t st);
// in int32 [n][n_in] -> out int8 [n][out_stride] (zero padded), argmax uint32 [n]; out / argmax may be null
void launch_relunorm(const int32_t *in, uint32_t n_in, int8_t *out, uint32_t out_stride, uint32_t *argmax, size_t n,
                     cudaStream_t st);
void launch_conv33relu(const int32_t *act, const int8_t *w, uint32_t n_w, uint32_t xy, uint32_t n_shift, int32_t *out,
                       size_t n, cudaStream_t st);
void launch_maxpool22(const int32_t *act, uint32_t xy, int32_t *out, size_t n, cudaStream_t st);
// fused CNN front-end (dll.c:64-80): images int8 [n][256] -> features int8 [n][feat_stride] after ReLUNorm over C*4
// returns false if the geometry is not the 16x16 / conv,conv,pool,conv,pool one
// frontend: 0 = tensor-core kernel when the shape is covered, else CUDA cores; 1 = CUDA cores (k_cnn_frontend16); 2 = tensor cores only
bool launch_cnn_frontend(const int8_t *images, const int8_t *w1, const int8_t *w2, const int8_t *w3, uint32_t channels,
                         uint32_t xy, int8_t *features, uint32_t feat_stride, size_t n, int sm_count, int frontend, int *d_err,
                         bool conv3_fits_u16, cudaStream_t st);
// the kernel launch_cnn_frontend runs for frontend and a model's shape (none: it returns false)
enum CnnFrontendKernel { kCnnFrontendNone, kCnnFrontendCudaCores, kCnnFrontendTensorCores };
CnnFrontendKernel cnn_frontend_kernel(uint32_t channels, uint32_t xy, int frontend);
// conv3_fits_u16: the pooled conv2 outputs (conv3's inputs) cannot exceed 65535 for this model's conv1 / conv2 weights
// (cnn_conv3_bound <= 65535, computed once per model): conv3 may then run on IDP.2A
long long cnn_conv3_bound(const int8_t *w1, const int8_t *w2, uint32_t channels);
bool cnn_frontend_tc_supported(uint32_t channels, uint32_t xy);

// same front-end with conv1 on wgmma and the depthwise tail fed from shared memory (cnn_wgmma.cu); false when the shape is not
// covered (channels not a multiple of 16, > 128, or geometry other than 16x16)
bool launch_cnn_frontend_tc(const int8_t *images, const int8_t *w1, const int8_t *w2, const int8_t *w3, uint32_t channels,
                            uint32_t xy, int8_t *features, uint32_t feat_stride, size_t n, int sm_count, int *d_err,
                            bool conv3_fits_u16, cudaStream_t st);

// emulation mode (BitNetMCU.py:420-535): normalisation rules of the reference's Python emulator, see generic_kernels.cu
void launch_relunorm_emul(const int32_t *in, uint32_t n_in, int level_shift, int8_t *out, uint32_t out_stride, size_t n, cudaStream_t st);
void launch_expand_image(const int8_t *img, int32_t *planes, uint32_t C, uint32_t elems, size_t n, cudaStream_t st);
void launch_conv_renorm(int32_t *planes, uint32_t elems_per_image, size_t n, cudaStream_t st);
void launch_i32_to_i8(const int32_t *in, uint32_t n_in, int8_t *out, uint32_t out_stride, size_t n, cudaStream_t st);
// the last layer's int32 accumulators [n][n_cls] -> float64 logits x 2^-level_shift and first-maximum labels (np.argmax); either
// output may be null
void launch_emul_logits(const int32_t *acc, uint32_t n_cls, int level_shift, double *logits, uint32_t *labels, size_t n, cudaStream_t st);
// top-k of rows [n][n_cls] (int32 or float64) -> classes uint32 [n][k] and scores [n][k] (may be null): the classes by value,
// highest first, ties to the lower class; 1 <= k <= n_cls
void launch_topk_rows(const int32_t *rows, uint32_t n_cls, uint32_t k, uint32_t *classes, int32_t *scores, size_t n, cudaStream_t st);
void launch_topk_rows(const double *rows, uint32_t n_cls, uint32_t k, uint32_t *classes, double *scores, size_t n, cudaStream_t st);

// 16-bit float image elements (BNM_FLOAT16 / BNM_BFLOAT16 of the header)
enum HalfFormat : uint32_t { kHalfFloat16 = 1, kHalfBFloat16 = 2 };

// The maximum of the input scaling's row maxima and of its 1e-5 floor: NaN if either operand is NaN, as NumPy's max and np.maximum
// are (fmaxf drops NaN).  With it a row holding any NaN gets a NaN scale, and one holding an infinity (and no NaN) a scale of 0;
// every product is then NaN or +-0, and a NaN product scales to 0 (what NaN.astype(np.int8) gives on x86-64 and AArch64): a row
// with any non-finite element scales to the all-zero int8 row, on every route.
__device__ __forceinline__ float fmax_nan(float a, float b) {
    float d;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(d) : "f"(a), "f"(b));
    return d;
}

// input quantisation ahead of the path (test_inference.py:140-141): float [n][elems] -> int8 [n][elems]
void launch_quantize_images(const float *in, uint32_t elems, int8_t *out, size_t n, cudaStream_t st);
// the same on 16-bit elements of format fmt [n][elems]: what the float32 kernel gives on them widened to float32
void launch_quantize_images(const uint16_t *in, HalfFormat fmt, uint32_t elems, int8_t *out, size_t n, cudaStream_t st);

// how a padded page's border pixels are made (section 13 of the header; the values of BNM_PAD_*): the fill value, the nearest
// edge pixel, or the mirror image about the edge pixel (which is not repeated)
enum PadMode : uint32_t { kPadConstant = 0, kPadReplicate = 1, kPadReflect = 2 };

// The 16x16 windows of a stack of planes (sections 9, 10, 12 and 13 of the header) of float32 elements (half == 0) or 16-bit ones
// of format half: plane p is image + p * plane_pitch elements, [height][pitch] on the device (16-byte aligned, pitch and plane_pitch
// multiples of 16 bytes), padded by top / left / right pixels (bottom ones only count in out_h) in pad_mode, its windows on an
// (stride_y, stride_x) grid of out_h x out_w over the padded plane.  Windows are numbered plane by plane, row-major within a
// plane: w = (p * out_h + r) * out_w + c.  Without padding every pad is 0.  Padded height and width fit in 32 bits.
struct WindowGrid {
    const void *image;
    uint32_t half;   // 0: float32 elements; kHalfFloat16 / kHalfBFloat16: 16-bit elements of that format
    uint32_t planes, height, width;
    size_t pitch, plane_pitch;
    uint32_t stride_y, stride_x, out_h, out_w;
    uint32_t top = 0, left = 0, right = 0, pad_mode = kPadConstant;   // pixels added above, left, right; a PadMode
    float pad_value = 0.0f;                                           // kPadConstant: the border's pixel value
};
// windows w0 .. w0 + n - 1 of g, each flattened row-major and scaled as launch_quantize_images scales an image (16-bit elements:
// widened to float32 first; border pixels made as pad_mode says) -> int8 [n][256] (16-byte aligned).  false when the kernel
// cannot get its shared memory.
bool launch_quantize_windows(const WindowGrid &g, size_t w0, size_t n, int8_t *out, cudaStream_t st);

// ---- scoring both engines (bnm_compare_engines_device): counts = uint64 {images, correct_c, correct_py, mismatches}, the layout of
// bnm_engine_counts.  A warp's counters: every lane of the warp calls add() with the row it holds (row = false: none); the flags
// are counted by ballot, kept in registers across the warp's rows, and flush() adds them with one 64-bit atomic per non-zero
// counter.  A truth value of n_classes or more never matches (no truth: pass ~0u).
struct EngineTally {
    uint32_t correct_c = 0, correct_py = 0, mismatches = 0;
    __device__ __forceinline__ void add(bool row, uint32_t label_c, uint32_t label_py, uint32_t truth, uint32_t n_classes) {
        const bool known = row && truth < n_classes;
        correct_c += __popc(__ballot_sync(0xffffffffu, known && label_c == truth));
        correct_py += __popc(__ballot_sync(0xffffffffu, known && label_py == truth));
        mismatches += __popc(__ballot_sync(0xffffffffu, row && label_c != label_py));
    }
    __device__ __forceinline__ void flush(unsigned long long *counts) const {
        if ((threadIdx.x & 31) != 0) return;
        if (correct_c) atomicAdd(&counts[1], (unsigned long long)correct_c);
        if (correct_py) atomicAdd(&counts[2], (unsigned long long)correct_py);
        if (mismatches) atomicAdd(&counts[3], (unsigned long long)mismatches);
    }
};
// the two engines' labels [n] (and truth [n] or null) -> counts += their tallies and images += n
void launch_engine_counts(const uint32_t *labels_c, const uint32_t *labels_py, const uint32_t *truth, size_t n, uint32_t n_classes,
                          unsigned long long *counts, cudaStream_t st);

// ---- fused wgmma FC chain (fc_wgmma.cu)
struct FcChainPlan;  // opaque, owned by the model
// verbose: print the plan's shapes now and every int8-form launch's wait decision (the model's BNM_VERBOSE at its creation)
FcChainPlan *fc_chain_plan_create(const FcLayerDev *layers, int n_layers, uint32_t in_bytes, int device, int sm_count, bool verbose,
                                  char *err, size_t err_len);
void fc_chain_plan_destroy(FcChainPlan *p);
// kFormInt8 launches: 0 plain launches, 1 programmatic dependent launch (inputs read after the previous kernel completed), 2 launches
// declared independent
void fc_chain_plan_set_overlap(FcChainPlan *p, int mode);
// The launch forms of a plan.  fc_wgmma.cu's form table (kForms) says what each is: its input (int8 rows [n][in_bytes] over
// TMA, device, 16B aligned; or float32 rows [n][in_bytes elements] with the input scaling of test_inference.py:140-141 fused
// into the load stage), its rule (the C engine's, the reference's Python emulator's, or both), its outputs and its kernel rows.
// A plan has every int8 form; the float-input forms only for models up to 64 wide with rows of up to 256 elements and up to
// 16 classes.  The emulator's logits are the last layer's accumulators x 2^-level_shift_of(its encoding), in float64.
// kFormFloat16, kFormEmulFloat16 and kFormEngines16 are kFormFloat, kFormEmulFloat and kFormEngines on 16-bit rows (HalfFormat):
// a plan has them exactly where it has those, and each gives what its float32 form gives on the rows widened to float32.
enum FcForm { kFormInt8, kFormFloat, kFormEmulFloat, kFormEmulInt8, kFormEngines, kFormTopK, kFormEmulTopK,
              kFormFloat16, kFormEmulFloat16, kFormEngines16, kFcForms };
bool fc_chain_has_form(const FcChainPlan *p, FcForm f);
// the kernel of a form the plan has, e.g. "fc_emul_i8_kernel<192,1,emul>"
const char *fc_chain_form_name(const FcChainPlan *p, FcForm f);
// the emulator's level scale of a layer is 2^level_shift_of(its encoding): 2 for 2bitsym / 4bitsym, else 1 (capi.cu)
int level_shift_of(int32_t enc);
// both engines' outputs besides `labels` (the C engine's): the emulator's labels uint32 [n], truth uint32 [n] and counts (each may
// be null; truth only with counts)
struct EngineOutputs {
    uint32_t *labels_py;
    const uint32_t *truth;
    unsigned long long *counts;
};
// top-k outputs: k (1 .. n_classes) classes uint32 [n][k], required, and their scores [n][k] (int32, float64 for the emulator) or null
struct TopKOutputs {
    uint32_t k;
    uint32_t *classes;
    void *scores;
};
// What a call writes, each buffer possibly null: logits (int32 [n][n_classes], float64 for the emulator) and labels uint32 [n],
// and gather: extra destination buffers every row is also stored to (peer memory), fused into the epilogue (the C engine on int8
// rows only).  Both engines' forms take labels and engines, no logits.  The top-k forms take topk alone, with k > 0; every other
// form takes none (k = 0).
struct FcOutputs {
    void *logits;
    uint32_t *labels;
    const GatherDst *gather;
    TopKOutputs topk;
    EngineOutputs engines;
};
// The capture state of a call's stream, read once per call (cudaStreamGetCaptureInfo): active while the stream is capturing into
// a graph, with the capture sequence's id (unique in the process).  A captured launch keeps its launch-overlap bookkeeping apart
// from the eager launches'.
struct StreamCapture {
    bool active = false;
    unsigned long long id = 0;
};
// one launch of form f on n images `in` -> out on st, whose capture state is cap.  0, or a negative code (-5: an output the form
// does not take, or a missing one; -6: the plan has no form f).  fed: `in` was written by a kernel of another kind that the same
// call launched just before into its scratch (k_quantize_windows, k_quantize_images, a CNN front-end); the launch keeps its grid-dependency wait and, as a launch of
// another kind, leaves the launch-overlap record empty, so the next int8 launch keeps its wait too.  in_format: the HalfFormat of
// a 16-bit form's rows, 0 for every other form.
int fc_chain_launch(FcChainPlan *p, FcForm f, const void *in, size_t n, const FcOutputs &out, cudaStream_t st, const StreamCapture &cap,
                    bool fed = false, uint32_t in_format = 0);
// the emulator's CNN front-end (BitNetMCU.py:435-445, 459-526) in one kernel: float32 images [n][256] -> int8 features
// [n][feat_stride], the (C, 2, 2) flatten; false when channels is 0 or more than kCnnEmulMaxChannels
constexpr uint32_t kCnnEmulMaxChannels = 128;
bool launch_cnn_emul_frontend(const float *images, const int8_t *w1, const int8_t *w2, const int8_t *w3, uint32_t channels,
                              int8_t *features, uint32_t feat_stride, size_t n, cudaStream_t st);
// the same front-end on images already scaled to int8 [n][256] (16-byte aligned rows, k_quantize_windows' output):
// k_cnn_emul_frontend_i8, the same features as the float kernel gives on the float images those rows were scaled from
bool launch_cnn_emul_frontend_i8(const int8_t *images, const int8_t *w1, const int8_t *w2, const int8_t *w3, uint32_t channels,
                                 int8_t *features, uint32_t feat_stride, size_t n, cudaStream_t st);

}  // namespace bnm
