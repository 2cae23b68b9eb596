// generic_kernels.cu -- CUDA-core kernels of the engine (any layer shape):
//   * weight pre-decode  : packed exportquant words -> dense int8 planes          (reference decode rules inference.c:96-201)
//   * processfclayer     : dp4a over the decoded planes, thread-per-image tile    (inference.c:88-208)
//   * ReLUNorm           : warp-per-row, shuffle max/argmax reduction             (inference.c:23-72)
//   * processconv33ReLU / processmaxpool22 batched                                (inference.c:238-277, 300-322)
//   * fused CNN front-end: conv,conv,pool,conv,pool per channel + ReLUNorm        (BitNetMCU_MNIST_dll.c:64-80)
//   * input scaling      : float rows, or the 16x16 windows of a float plane (shared band), to int8 rows (test_inference.py:140-141)
// These are the layer-by-layer path (BNM_PATH_LAYERS) and the front half of every CNN model; the fused
// wgmma FC chain lives in fc_wgmma.cu.
#include <algorithm>
#include <map>
#include <mutex>
#include <utility>

#include "kernels.h"

namespace bnm {

// ------------------------------------------------------------------------------------------------
// weight decode
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ int decode_weight(const void *packed, int32_t enc, uint32_t n_in, uint32_t o, uint32_t k, int nf4_ext) {
    const uint32_t *w32 = static_cast<const uint32_t *>(packed);
    switch (enc) {
    case 1: {  // Binary: bit set -> +1, clear -> -1 (inference.c:96-104); first weight in the MSB
        uint32_t w = w32[(size_t)o * ((n_in + 31) / 32) + k / 32];
        return ((w >> (31 - (k & 31))) & 1u) ? 1 : -1;
    }
    case 2: {  // 2bitsym: sign bit + magnitude bit -> +-1, +-3 (inference.c:105-115)
        uint32_t c = (w32[(size_t)o * ((n_in + 15) / 16) + k / 16] >> (30 - 2 * (k & 15))) & 3u;
        int mag = 1 + 2 * (int)(c & 1u);
        return (c & 2u) ? -mag : mag;
    }
    case 4: case 12: case 20: case 36: {
        uint32_t c = (w32[(size_t)o * ((n_in + 7) / 8) + k / 8] >> (28 - 4 * (k & 7))) & 15u;
        if (enc == 4) { int mag = 2 * (int)(c & 7u) + 1; return (c & 8u) ? -mag : mag; }           // inference.c:156-168
        if (enc == 12) return (int)(c ^ 8u) - 8;                                                   // two's complement nibble, 169-178
        if (enc == 20) { int mag = 1 << (c & 7u); return (c & 8u) ? -mag : mag; }                  // FP130, 190-201
        if (!nf4_ext) return 0;                                                                    // NF4: inference.c:202 -> zeros
        const int lut[16] = {-127, -88, -67, -50, -36, -23, -12, 0, 10, 20, 31, 43, 56, 71, 92, 127};
        return lut[c];
    }
    case 16: {  // 8-bit two's complement (inference.c:179-188)
        uint32_t c = (w32[(size_t)o * ((n_in + 3) / 4) + k / 4] >> (24 - 8 * (k & 3))) & 255u;
        return (int)(int8_t)c;
    }
    case 64: {  // Ternary: 10 trits per uint16, repeated *3 extraction (inference.c:116-136)
        const uint16_t *w16 = static_cast<const uint16_t *>(packed);
        uint32_t c = w16[(size_t)o * (n_in / 10) + k / 10];
        int w = 0;
        for (uint32_t j = 0; j <= k % 10; j++) {
            c *= 3u;
            w = (c & 0x20000u) ? 0 : ((c & 0x10000u) ? -1 : 1);
            c &= 0xFFFFu;
        }
        return w;
    }
    default:
        return 0;  // unsupported id: silent zeros (inference.c:202)
    }
}

__global__ void k_decode_fc(const void *packed, int32_t enc, uint32_t n_in, uint32_t n_out, uint32_t k_pad, uint32_t n_pad,
                            int8_t *dense_a, int8_t *dense_b, int nf4_ext, int *flag) {
    size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)k_pad * n_pad) return;
    uint32_t o = idx / k_pad, k = idx % k_pad;
    int w = (o < n_out && k < n_in) ? decode_weight(packed, enc, n_in, o, k, nf4_ext) : 0;
    int a = max(-128, min(127, w));   // plane A
    int b = w - a;                    // plane B: only FP130's +128 leaves a residual (+1)
    dense_a[idx] = (int8_t)a;
    dense_b[idx] = (int8_t)b;
    if (b != 0) atomicOr(flag, 1);
}

// quad layout for the dp4a kernel: q[(o/4)*(k_pad/4) + k4] = {w(o,k4), w(o+1,k4), w(o+2,k4), w(o+3,k4)}
__global__ void k_make_quads(const int8_t *dense, uint32_t k_pad, uint32_t n_pad, int4 *quads) {
    size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t k4n = k_pad / 4;
    if (idx >= (size_t)(n_pad / 4) * k4n) return;
    uint32_t og = idx / k4n, k4 = idx % k4n;
    const uint32_t *d = reinterpret_cast<const uint32_t *>(dense);
    int4 q;
    q.x = d[(size_t)(og * 4 + 0) * k4n + k4];
    q.y = d[(size_t)(og * 4 + 1) * k4n + k4];
    q.z = d[(size_t)(og * 4 + 2) * k4n + k4];
    q.w = d[(size_t)(og * 4 + 3) * k4n + k4];
    quads[idx] = q;
}

void launch_decode_fc(const void *d_packed, int32_t enc, uint32_t n_in, uint32_t n_out, uint32_t k_pad, uint32_t n_pad,
                      int8_t *dense_a, int8_t *dense_b, int4 *quad_a, int4 *quad_b, int nf4_extension, int *d_flag,
                      cudaStream_t st) {
    size_t total = (size_t)k_pad * n_pad;
    k_decode_fc<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(d_packed, enc, n_in, n_out, k_pad, n_pad, dense_a, dense_b,
                                                                nf4_extension, d_flag);
    size_t nq = (size_t)(n_pad / 4) * (k_pad / 4);
    k_make_quads<<<(unsigned)((nq + 255) / 256), 256, 0, st>>>(dense_a, k_pad, n_pad, quad_a);
    k_make_quads<<<(unsigned)((nq + 255) / 256), 256, 0, st>>>(dense_b, k_pad, n_pad, quad_b);
}

// ------------------------------------------------------------------------------------------------
// processfclayer on CUDA cores: 128 images per CTA (one per thread), activations staged in smem with an
// odd word stride (conflict-free), weights read as warp-uniform 128-bit loads, 4 outputs per pass (dp4a).
// A row holds act_valid bytes, then zeros up to k_pad (the reference's memset layer_in).  Rows of 4-aligned
// address and stride (act_valid is then a multiple of 4) stage as words; any other row -- a first layer on
// images of img_bytes % 4 != 0, e.g. a 130-byte Ternary row -- byte by byte, never past its own last byte.
// ------------------------------------------------------------------------------------------------
template <bool HAS_B>
__global__ void __launch_bounds__(128) k_fc_dp4a(const int8_t *__restrict__ act, uint32_t act_stride, uint32_t act_valid,
                                                  const int4 *__restrict__ qa, const int4 *__restrict__ qb, uint32_t k4n,
                                                  uint32_t n_out, uint32_t n_pad, int32_t *__restrict__ out, size_t n) {
    extern __shared__ uint32_t s_act[];  // [128][k4n + 1]
    const uint32_t tid = threadIdx.x;
    const size_t img0 = (size_t)blockIdx.x * 128;
    const uint32_t stride = k4n + 1;
    const bool words = (((uintptr_t)act | act_stride) & 3) == 0;
    for (uint32_t idx = tid; idx < 128 * k4n; idx += 128) {
        uint32_t im = idx / k4n, k4 = idx % k4n;
        uint32_t v = 0;
        if (img0 + im < n && k4 * 4 < act_valid) {
            const int8_t *p = act + (img0 + im) * act_stride + k4 * 4;
            if (words) {
                v = *reinterpret_cast<const uint32_t *>(p);
            } else {
#pragma unroll
                for (uint32_t j = 0; j < 4; j++)
                    if (k4 * 4 + j < act_valid) v |= (uint32_t)(uint8_t)p[j] << (8 * j);
            }
        }
        s_act[im * stride + k4] = v;
    }
    __syncthreads();
    if (img0 + tid >= n) return;
    const uint32_t *a = s_act + tid * stride;
    int32_t *o = out + (img0 + tid) * n_out;
    for (uint32_t og = 0; og < n_pad / 4; og++) {
        int acc0 = 0, acc1 = 0, acc2 = 0, acc3 = 0;
        const int4 *wa = qa + (size_t)og * k4n;
        const int4 *wb = qb + (size_t)og * k4n;
#pragma unroll 4
        for (uint32_t k4 = 0; k4 < k4n; k4++) {
            int av = (int)a[k4];
            int4 w = __ldg(wa + k4);
            acc0 = __dp4a(av, w.x, acc0);
            acc1 = __dp4a(av, w.y, acc1);
            acc2 = __dp4a(av, w.z, acc2);
            acc3 = __dp4a(av, w.w, acc3);
            if (HAS_B) {
                int4 v = __ldg(wb + k4);
                acc0 = __dp4a(av, v.x, acc0);
                acc1 = __dp4a(av, v.y, acc1);
                acc2 = __dp4a(av, v.z, acc2);
                acc3 = __dp4a(av, v.w, acc3);
            }
        }
        uint32_t ob = og * 4;
        if (ob + 0 < n_out) o[ob + 0] = acc0;
        if (ob + 1 < n_out) o[ob + 1] = acc1;
        if (ob + 2 < n_out) o[ob + 2] = acc2;
        if (ob + 3 < n_out) o[ob + 3] = acc3;
    }
}

bool launch_fc_dp4a(const int8_t *act, uint32_t act_stride, const FcLayerDev &L, int32_t *out, size_t n, cudaStream_t st) {
    if (n == 0) return true;
    uint32_t k4n = L.k_pad / 4;
    size_t smem = (size_t)128 * (k4n + 1) * 4;
    if (smem > 227 * 1024) return false;   // 128 staged rows of more than ~1.8k inputs do not fit an SM
    unsigned grid = (unsigned)((n + 127) / 128);
    uint32_t valid = act_stride < L.k_pad ? act_stride : L.k_pad;
    auto *kernel = L.dense_b ? k_fc_dp4a<true> : k_fc_dp4a<false>;
    if (!raise_smem_limit((const void *)kernel, smem)) return false;
    kernel<<<grid, 128, smem, st>>>(act, act_stride, valid, L.quad_a, L.dense_b ? L.quad_b : L.quad_a, k4n, L.n_out, L.n_pad, out, n);
    return true;
}

bool raise_smem_limit(const void *kernel, size_t bytes) {
    static std::mutex mu;   // a concurrent raise to fewer bytes must not undo one to more
    static std::map<std::pair<int, const void *>, size_t> known;   // (device, kernel) -> a limit it is known to have
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return false; }
    std::lock_guard<std::mutex> lock(mu);
    size_t &limit = known[{dev, kernel}];
    if (bytes <= limit) return true;
    cudaFuncAttributes a;
    cudaError_t e = cudaFuncGetAttributes(&a, kernel);
    if (e == cudaSuccess && bytes > (size_t)a.maxDynamicSharedSizeBytes)
        e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) {
        cudaGetLastError();   // not sticky: leave no stale error behind for the caller's launch check
        return false;
    }
    limit = std::max(bytes, (size_t)a.maxDynamicSharedSizeBytes);
    return true;
}

// ------------------------------------------------------------------------------------------------
// ReLUNorm: one warp per row.  argmax = first maximum (strict '>' from -INT32_MAX / position 255).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t relunorm_shift(int32_t max_val) {
    // bit length of (max >> 7) (inference.c:41-47); a negative maximum zeroes every output anyway
    if (max_val <= 0) return 0;
    uint32_t scale = (uint32_t)(max_val >> 7);
    return scale ? 32u - (uint32_t)__clz((int)scale) : 0u;
}

__global__ void __launch_bounds__(256) k_relunorm(const int32_t *__restrict__ in, uint32_t n_in, int8_t *__restrict__ out,
                                                   uint32_t out_stride, uint32_t *__restrict__ argmax, size_t n) {
    const uint32_t lane = threadIdx.x & 31;
    const size_t row = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n) return;
    const int32_t *x = in + row * n_in;
    int32_t best = -INT32_MAX;
    uint32_t pos = 255;
    for (uint32_t i = lane; i < n_in; i += 32) {
        int32_t v = x[i];
        if (v > best) { best = v; pos = i; }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        int32_t ov = __shfl_xor_sync(0xffffffffu, best, off);
        uint32_t op = __shfl_xor_sync(0xffffffffu, pos, off);
        if (ov > best || (ov == best && op < pos)) { best = ov; pos = op; }
    }
    if (argmax && lane == 0) argmax[row] = pos;
    if (!out) return;
    const uint32_t shift = relunorm_shift(best);
    const int32_t rounding = (int32_t)((1u << shift) >> 1);
    int8_t *y = out + row * out_stride;
    for (uint32_t i = lane; i < out_stride; i += 32) {
        int32_t r = 0;
        if (i < n_in) {
            int32_t v = x[i];
            r = v < 0 ? 0 : min(127, (v + rounding) >> shift);
        }
        y[i] = (int8_t)r;
    }
}

void launch_relunorm(const int32_t *in, uint32_t n_in, int8_t *out, uint32_t out_stride, uint32_t *argmax, size_t n,
                     cudaStream_t st) {
    if (n == 0) return;
    k_relunorm<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(in, n_in, out, out_stride, argmax, n);
}

// ------------------------------------------------------------------------------------------------
// Input quantisation, the step right before the path (SURVEY.md 8f rank 3): test_inference.py:140-141 /
// BitNetMCU.py:435-436:  scale = 127 / max(max|x|, 1e-5);  q = round_half_even(x * scale).clip(-128, 127)  in float32.
// One warp per image; every operation is a single correctly rounded IEEE float32 op (no FMA contraction), so the result
// is bit-identical to the NumPy expression.  The maxima propagate NaN (fmax_nan, kernels.h) and a NaN product scales to 0, as
// NumPy's expression followed by .astype(np.int8) does: a row with any NaN or infinity becomes the all-zero row.
// ------------------------------------------------------------------------------------------------
// scale of an image whose largest |x| is absmax, and one pixel scaled with it (k_quantize_images, k_cnn_emul_frontend)
__device__ __forceinline__ float quant_scale(float absmax) { return __fdiv_rn(127.0f, fmax_nan(absmax, 1e-5f)); }
__device__ __forceinline__ int quant_pixel(float x, float scale) {
    // np.round (half to even) with cvt.rni, which gives 0 for NaN and saturates at the int32 range, then .clip(-128, 127)
    return min(max(__float2int_rn(__fmul_rn(x, scale)), -128), 127);
}

__global__ void __launch_bounds__(256) k_quantize_images(const float *__restrict__ in, uint32_t elems, int8_t *__restrict__ out, size_t n) {
    const uint32_t lane = threadIdx.x & 31;
    const size_t img = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (img >= n) return;
    const float *x = in + img * elems;
    float m = 0.0f;
    for (uint32_t i = lane; i < elems; i += 32) m = fmax_nan(m, fabsf(x[i]));
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) m = fmax_nan(m, __shfl_xor_sync(0xffffffffu, m, off));
    const float scale = quant_scale(m);
    int8_t *q = out + img * elems;
    for (uint32_t i = lane; i < elems; i += 32) q[i] = (int8_t)quant_pixel(x[i], scale);
}

void launch_quantize_images(const float *in, uint32_t elems, int8_t *out, size_t n, cudaStream_t st) {
    if (n == 0 || elems == 0) return;
    k_quantize_images<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(in, elems, out, n);
}

// The same scaling on 16-bit elements of format kFmt: each element widened exactly to float32 (bfloat16: the top half of a
// float32; float16: cvt.f32.f16), then the float32 kernel's steps, row maximum in float32 included.  Any row length.
template <HalfFormat kFmt> __device__ __forceinline__ float widen_half(uint16_t h) {
    if (kFmt == kHalfBFloat16) return __uint_as_float((uint32_t)h << 16);
    float f;
    asm("cvt.f32.f16 %0, %1;" : "=f"(f) : "h"(h));
    return f;
}
template <HalfFormat kFmt>
__global__ void __launch_bounds__(256) k_quantize_images(const uint16_t *__restrict__ in, uint32_t elems, int8_t *__restrict__ out, size_t n) {
    const uint32_t lane = threadIdx.x & 31;
    const size_t img = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (img >= n) return;
    const uint16_t *x = in + img * elems;
    float m = 0.0f;
    for (uint32_t i = lane; i < elems; i += 32) m = fmax_nan(m, fabsf(widen_half<kFmt>(x[i])));
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) m = fmax_nan(m, __shfl_xor_sync(0xffffffffu, m, off));
    const float scale = quant_scale(m);
    int8_t *q = out + img * elems;
    for (uint32_t i = lane; i < elems; i += 32) q[i] = (int8_t)quant_pixel(widen_half<kFmt>(x[i]), scale);
}

void launch_quantize_images(const uint16_t *in, HalfFormat fmt, uint32_t elems, int8_t *out, size_t n, cudaStream_t st) {
    if (n == 0 || elems == 0) return;
    if (fmt == kHalfBFloat16) k_quantize_images<kHalfBFloat16><<<(unsigned)((n + 7) / 8), 256, 0, st>>>(in, elems, out, n);
    else k_quantize_images<kHalfFloat16><<<(unsigned)((n + 7) / 8), 256, 0, st>>>(in, elems, out, n);
}

// ------------------------------------------------------------------------------------------------
// Window scan (bnm_infer_windows_device_f32, bnm_scan_windows_device and the other stacked entries, float32 or 16-bit, padded or
// not): the 16x16 windows of a stack of planes, each scaled as k_quantize_images scales an image, into int8 rows [n][256].  The
// window rows of the stack are numbered plane by plane, and a CTA takes a run of up to kWinCta windows of one window row.  They
// share their 16 pixel rows, and the columns they span (at most kWinBox) are loaded ONCE into shared memory as a float32 band, row
// by row with coalesced loads (16-bit elements widened on the way: the plane's element kind is a runtime field, so one function
// serves all three): each pixel of the band comes from L2 / HBM once per band, not once per window covering it.  Padding (section
// 13) is runtime fields too, and only changes where a band element comes from: a band wholly on the page takes the plain load,
// a band reaching into the border maps each of its rows and columns to the page's (clamped or mirrored) or to the fill value.
// From the band: every column's
// max |x| over the 16 rows, then per window (one thread each) the max of its 16 columns -- a 16-wide sliding max; both carry NaN,
// so a window covering a NaN or infinite pixel is the all-zero row and its neighbours are untouched -- the scale,
// and its 256 pixels into a staging row padded to 272 bytes (16-byte stores of one quarter-warp then hit distinct banks).  The
// CTA's rows are consecutive windows, so they leave as one contiguous run of coalesced 16-byte stores.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kWinCta = 128, kWinBox = 256, kWinStage = 272;
constexpr size_t kWinSmem = 16 * kWinBox * 4 + kWinBox * 4 + kWinCta * kWinStage;   // band, column maxima, staging

struct WindowRun {
    const void *image;
    uint32_t half;              // 0: float32 planes; else the HalfFormat of 16-bit planes
    size_t pitch, plane_pitch;  // elements between rows, between planes
    uint32_t height, width;     // of the page
    uint32_t top, left, pad_w;  // pixels added above and left; the padded width (the page's when unpadded)
    uint32_t pad_mode;          // a PadMode
    float pad_value;            // kPadConstant: the border's pixel value
    uint32_t stride_y, stride_x, out_h, out_w;   // the grid over the padded page
    uint32_t per_cta, chunks;   // windows per CTA (per_cta columns of the grid, one box); CTAs per window row
    uint32_t box_w;             // band width in pixels
    size_t run0;                // the pass's first run of windows: run g covers window row g / chunks of the stack (row
                                // g / chunks % out_h of plane g / chunks / out_h), columns (g % chunks) * per_cta ..
    size_t w0, n;               // the pass: windows w0 .. w0 + n - 1
    int8_t *out;                // [n][256]
};

// a band element as float32: float32 as it is, a 16-bit one widened exactly (widen_half)
template <HalfFormat kFmt> __device__ __forceinline__ float band_elem(float x) { return x; }
template <HalfFormat kFmt> __device__ __forceinline__ float band_elem(uint16_t h) { return widen_half<kFmt>(h); }

// the band of 16 rows from src (the first row's column x0, rows pitch elements apart) into band [16][box_w], cols columns of
// pixels and zeros past them (a zero element widens to +0.0); kFmt: the format of 16-bit elements (unused for float32 ones).  A
// column's rows go in two groups of 8 loads, each issued before its first store (measured on float32 planes: no slower than the
// float32-only loop this replaced; all 16 at once was 0.4% slower on 4096-wide pages at stride 1)
template <HalfFormat kFmt = kHalfFloat16, class T>
__device__ __forceinline__ void load_band(float *band, const T *__restrict__ src, size_t pitch, uint32_t box_w, uint32_t cols) {
    for (uint32_t x = threadIdx.x; x < box_w; x += blockDim.x) {
#pragma unroll
        for (int y0 = 0; y0 < 16; y0 += 8) {
            T v[8];
#pragma unroll
            for (int y = 0; y < 8; y++) v[y] = x < cols ? __ldg(src + (size_t)(y0 + y) * pitch + x) : T(0);
#pragma unroll
            for (int y = 0; y < 8; y++) band[(y0 + y) * box_w + x] = band_elem<kFmt>(v[y]);
        }
    }
}

// the page index of padded index i (counted from the page's first pixel) on a side of n pixels: i itself on the page, else the
// edge pixel (replicate), its mirror image about the edge pixel (reflect: a pad is < n, so one reflection lands on the page), or
// -1 for the fill value (constant)
__device__ __forceinline__ long long pad_index(long long i, uint32_t n, uint32_t mode) {
    if (i >= 0 && i < n) return i;
    if (mode == kPadReplicate) return i < 0 ? 0 : (long long)n - 1;
    if (mode == kPadReflect) return i < 0 ? -i : 2 * ((long long)n - 1) - i;
    return -1;
}

// load_band for a band that reaches into the border: band row y is page row rows[y] (its element offset in the stack, -1 for the
// fill value) and band column x page column pad_index(cx + x), cols columns of pixels and zeros past them (past the padded width,
// never read by a window).  Only page pixels are read; the fill value goes into the band as it is
template <HalfFormat kFmt = kHalfFloat16, class T>
__device__ __forceinline__ void load_band_padded(float *band, const T *__restrict__ image, const long long *rows, long long cx,
                                                 uint32_t width, uint32_t mode, float value, uint32_t box_w, uint32_t cols) {
    for (uint32_t x = threadIdx.x; x < box_w; x += blockDim.x) {
        const long long c = x < cols ? pad_index(cx + x, width, mode) : -1;
        const float fill = x < cols ? value : 0.0f;
#pragma unroll 4
        for (int y = 0; y < 16; y++) {
            const long long o = rows[y];
            band[y * box_w + x] = c < 0 || o < 0 ? fill : band_elem<kFmt>(__ldg(image + o + c));
        }
    }
}

__global__ void __launch_bounds__(kWinCta) k_quantize_windows(const WindowRun a) {
    extern __shared__ __align__(16) uint8_t smem[];
    float *band = reinterpret_cast<float *>(smem);        // [16][box_w]
    float *colmax = band + 16 * kWinBox;                  // [box_w]
    uint8_t *stage = reinterpret_cast<uint8_t *>(colmax + kWinBox);   // [per_cta][kWinStage]
    const size_t g = a.run0 + blockIdx.x;   // CTAs cover the runs the pass touches, and no others
    const size_t row = g / a.chunks, p = row / a.out_h;   // the window row in the stack, its plane
    const uint32_t r = (uint32_t)(row - p * a.out_h), c0 = (uint32_t)(g % a.chunks) * a.per_cta;
    const size_t first = row * a.out_w + c0;   // the CTA's windows first .. first + per_cta - 1, clipped to the row and the pass
    const size_t lo = max(first, a.w0), hi = min(first + min(a.per_cta, a.out_w - c0), a.w0 + a.n);
    if (lo >= hi) return;
    // the band: padded rows r * stride_y .. + 15 of plane p, padded columns x0 .. x0 + box_w - 1 (zeros past the padded width,
    // never read by a window); the plane's offset is 64-bit, past 2^31 elements in a stack of large pages.  16-bit planes are
    // widened to float32 here, so everything after the band load is the float32 kernel's
    const uint32_t x0 = c0 * a.stride_x, cols = min(a.box_w, a.pad_w - x0);
    const long long y0 = (long long)r * a.stride_y - a.top, cx = (long long)x0 - a.left;   // the band's first pixel on the page
    if (y0 >= 0 && y0 + 16 <= a.height && cx >= 0 && cx + cols <= a.width) {   // wholly on the page: every unpadded CTA
        const size_t at = p * a.plane_pitch + (size_t)y0 * a.pitch + (size_t)cx;   // elements
        if (a.half == kHalfFloat16) load_band<kHalfFloat16>(band, static_cast<const uint16_t *>(a.image) + at, a.pitch, a.box_w, cols);
        else if (a.half == kHalfBFloat16) load_band<kHalfBFloat16>(band, static_cast<const uint16_t *>(a.image) + at, a.pitch, a.box_w, cols);
        else load_band(band, static_cast<const float *>(a.image) + at, a.pitch, a.box_w, cols);
    } else {   // a border CTA: its 16 rows mapped once, into colmax's space (not written before the band is complete)
        long long *rows = reinterpret_cast<long long *>(colmax);
        if (threadIdx.x < 16) {
            const long long y = pad_index(y0 + threadIdx.x, a.height, a.pad_mode);
            rows[threadIdx.x] = y < 0 ? -1 : (long long)(p * a.plane_pitch + (size_t)y * a.pitch);
        }
        __syncthreads();
        if (a.half == kHalfFloat16)
            load_band_padded<kHalfFloat16>(band, static_cast<const uint16_t *>(a.image), rows, cx, a.width, a.pad_mode, a.pad_value, a.box_w, cols);
        else if (a.half == kHalfBFloat16)
            load_band_padded<kHalfBFloat16>(band, static_cast<const uint16_t *>(a.image), rows, cx, a.width, a.pad_mode, a.pad_value, a.box_w, cols);
        else load_band_padded(band, static_cast<const float *>(a.image), rows, cx, a.width, a.pad_mode, a.pad_value, a.box_w, cols);
    }
    __syncthreads();
    for (uint32_t x = threadIdx.x; x < a.box_w; x += blockDim.x) {
        float m = 0.0f;
#pragma unroll
        for (int y = 0; y < 16; y++) m = fmax_nan(m, fabsf(band[y * a.box_w + x]));
        colmax[x] = m;
    }
    __syncthreads();
    const uint32_t j = threadIdx.x;   // this thread's window: first + j
    if (first + j >= lo && first + j < hi) {
        const uint32_t xj = j * a.stride_x;
        float m = 0.0f;
#pragma unroll
        for (int k = 0; k < 16; k++) m = fmax_nan(m, colmax[xj + k]);
        const float scale = quant_scale(m);
#pragma unroll 4
        for (int y = 0; y < 16; y++) {
            const float *px = band + y * a.box_w + xj;
            uint32_t v[4];
#pragma unroll
            for (int q = 0; q < 4; q++)
                v[q] = (uint32_t)(quant_pixel(px[4 * q], scale) & 0xff) | (uint32_t)(quant_pixel(px[4 * q + 1], scale) & 0xff) << 8 |
                       (uint32_t)(quant_pixel(px[4 * q + 2], scale) & 0xff) << 16 | (uint32_t)(quant_pixel(px[4 * q + 3], scale) & 0xff) << 24;
            *reinterpret_cast<uint4 *>(stage + j * kWinStage + 16 * y) = make_uint4(v[0], v[1], v[2], v[3]);
        }
    }
    __syncthreads();
    const uint32_t s0 = (uint32_t)(lo - first), chunks = (uint32_t)(hi - lo) * 16;   // 16-byte chunks of the CTA's rows
    uint4 *dst = reinterpret_cast<uint4 *>(a.out + (lo - a.w0) * 256);
    for (uint32_t e = threadIdx.x; e < chunks; e += blockDim.x)
        dst[e] = *reinterpret_cast<const uint4 *>(stage + (s0 + e / 16) * kWinStage + (e % 16) * 16);
}

bool launch_quantize_windows(const WindowGrid &g, size_t w0, size_t n, int8_t *out, cudaStream_t st) {
    if (n == 0) return true;
    WindowRun a;
    a.image = g.image;
    a.half = g.half;
    a.pitch = g.pitch;
    a.plane_pitch = g.plane_pitch;
    a.height = g.height;
    a.width = g.width;
    a.top = g.top;
    a.left = g.left;
    a.pad_w = g.width + g.left + g.right;
    a.pad_mode = g.pad_mode;
    a.pad_value = g.pad_value;
    a.stride_y = g.stride_y;
    a.stride_x = g.stride_x;
    a.out_h = g.out_h;
    a.out_w = g.out_w;
    a.per_cta = std::min<uint32_t>({kWinCta, (kWinBox - 16) / g.stride_x + 1, g.out_w});
    a.chunks = (g.out_w + a.per_cta - 1) / a.per_cta;
    a.box_w = (a.per_cta - 1) * g.stride_x + 16;
    auto run_of = [&](size_t w) { return w / g.out_w * a.chunks + w % g.out_w / a.per_cta; };
    a.run0 = run_of(w0);
    a.w0 = w0;
    a.n = n;
    a.out = out;
    const size_t runs = run_of(w0 + n - 1) - a.run0 + 1;
    if (!raise_smem_limit((const void *)k_quantize_windows, kWinSmem)) return false;
    k_quantize_windows<<<(unsigned)runs, kWinCta, kWinSmem, st>>>(a);
    return true;
}

// ------------------------------------------------------------------------------------------------
// Emulation mode: the normalisation rules of the reference's Python emulator QuantizedModel.inference_quantized
// (/root/reference/BitNetMCU.py:420-535) instead of the C engine's -- SURVEY.md 8f rank 4.  The emulator works on weight LEVELS
// (4bitsym +-0.5..+-7.5, 2bitsym +-0.5/+-1.5: half the engine's integer weights) in float64; every quantity below is an exact dyadic
// rational, so the integer restatement reproduces it bit for bit:
//   BitLinear (452-457): conv = acc / level_scale;  rescale = 2^floor(log2(127 / max(conv.max, 1e-5)));
//                        out = round_half_even(conv * rescale).clip(0, 127)
//   BitConv2d (495-499): out = round_half_even(relu(conv) * (127.0 / max over the image)).clip(0, 127)   (float64, as NumPy)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_relunorm_emul(const int32_t *__restrict__ in, uint32_t n_in, int level_shift, int8_t *__restrict__ out,
                                                        uint32_t out_stride, size_t n) {
    const uint32_t lane = threadIdx.x & 31;
    const size_t row = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n) return;
    const int32_t *x = in + row * n_in;
    int32_t m = INT32_MIN;
    for (uint32_t i = lane; i < n_in; i += 32) m = max(m, x[i]);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, off));
    // k = floor(log2(127 * level_scale / m)): the largest k with m * 2^k <= 127 * level_scale (k < 0: m <= (127 * level_scale) << -k)
    int e = 0;
    if (m > 0) {
        const long long t = 127ll << level_shift;
        int k = 0;
        if ((long long)m <= t) { while (((long long)m << (k + 1)) <= t) k++; }
        else { k = -1; while ((long long)m > (t << -k)) k--; }
        e = k - level_shift;   // out = round_half_even(acc * 2^e)
    }
    int8_t *y = out + row * out_stride;
    for (uint32_t i = lane; i < out_stride; i += 32) {
        int r = 0;
        if (i < n_in && m > 0) {
            const int32_t v = x[i];
            if (v > 0) {
                long long q;
                if (e >= 0) q = (long long)v << e;
                else {
                    const int sft = -e;
                    q = (long long)v >> sft;
                    const long long rem = (long long)v & ((1ll << sft) - 1), half = 1ll << (sft - 1);
                    if (rem > half || (rem == half && (q & 1))) q++;   // np.round: half to even
                }
                r = (int)(q > 127 ? 127 : q);
            }
        }
        y[i] = (int8_t)r;
    }
}

// images int8 [n][256] -> int32 planes [(image, channel)][256], the copy loop of dll.c:68-70 for every channel
__global__ void k_expand_image(const int8_t *__restrict__ img, int32_t *__restrict__ planes, uint32_t C, uint32_t elems, size_t n) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n * C * elems) return;
    const size_t item = idx / elems;
    planes[idx] = img[(item / C) * elems + idx % elems];
}

// BitConv2d's renormalisation of one ReLU'd conv output v >= 0 of an image whose conv outputs have the maximum m:
// round_half_even(v * (127.0 / m)).clip(0, 127), float64 like NumPy (k_conv_renorm, k_cnn_emul_frontend).  m <= 0 (every output
// is zero): NumPy divides by zero there (nan); the scale 0 defines the result as zeros.
__device__ __forceinline__ double conv_renorm_scale(int m) { return m > 0 ? 127.0 / (double)m : 0.0; }
__device__ __forceinline__ int conv_renorm(int v, double scale) {
    return (int)fmin(fmax(rint(__dmul_rn((double)v, scale)), 0.0), 127.0);
}

// per image: v = round_half_even(v * (127.0 / max)).clip(0, 127) over its C * H * W conv outputs (already >= 0), float64 like NumPy
__global__ void __launch_bounds__(256) k_conv_renorm(int32_t *__restrict__ planes, uint32_t elems, size_t n) {
    __shared__ int s_max[8];
    int32_t *p = planes + (size_t)blockIdx.x * elems;
    int m = 0;
    for (uint32_t i = threadIdx.x; i < elems; i += 256) m = max(m, p[i]);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, off));
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = m;
    __syncthreads();
    m = s_max[0];
#pragma unroll
    for (int w = 1; w < 8; w++) m = max(m, s_max[w]);
    if (m <= 0) return;   // all-zero conv output: already the result (conv_renorm_scale)
    const double scale = conv_renorm_scale(m);
    for (uint32_t i = threadIdx.x; i < elems; i += 256) p[i] = conv_renorm(p[i], scale);
}

__global__ void k_i32_to_i8(const int32_t *__restrict__ in, uint32_t n_in, int8_t *__restrict__ out, uint32_t out_stride, size_t n) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n * out_stride) return;
    const size_t row = idx / out_stride;
    const uint32_t c = idx % out_stride;
    out[idx] = c < n_in ? (int8_t)in[row * n_in + c] : (int8_t)0;
}

// one thread per image: logits = acc x 2^-level_shift (exact in float64), label = first maximum
__global__ void k_emul_logits(const int32_t *__restrict__ acc, uint32_t n_cls, double scale, double *__restrict__ logits,
                              uint32_t *__restrict__ labels, size_t n) {
    const size_t row = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n) return;
    const int32_t *x = acc + row * n_cls;
    int32_t best = x[0];
    uint32_t pos = 0;
    for (uint32_t c = 0; c < n_cls; c++) {
        const int32_t v = x[c];
        if (logits) logits[row * n_cls + c] = (double)v * scale;
        if (v > best) { best = v; pos = c; }
    }
    if (labels) labels[row] = pos;
}

void launch_emul_logits(const int32_t *acc, uint32_t n_cls, int level_shift, double *logits, uint32_t *labels, size_t n, cudaStream_t st) {
    if (n && n_cls) k_emul_logits<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(acc, n_cls, level_shift ? 0.5 : 1.0, logits, labels, n);
}

// Top-k of the layer-by-layer routes: one warp per row, k rounds.  Round t takes the first maximum of the columns ranked after
// round t - 1's pick (v, p) -- x < v, or x == v at a column > p; round 0 takes every column -- by a strided scan and a shfl.xor
// reduction, as fc_topk_kernel's epilogue does over its quads.  Lane t % 32 keeps round t's pick and stores it with the others
// after every 32nd and the last round.
template <class T>
__global__ void __launch_bounds__(256) k_topk_rows(const T *__restrict__ rows, uint32_t n_cls, uint32_t k, uint32_t *__restrict__ classes,
                                                   T *__restrict__ scores, size_t n) {
    constexpr uint32_t kNone = 0xffffffffu;
    const uint32_t lane = threadIdx.x & 31;
    const size_t row = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= n) return;
    const T *x = rows + row * n_cls;
    T v = 0, my_score = 0;
    uint32_t p = kNone, my_cls = 0;
    for (uint32_t t = 0; t < k; t++) {
        T best = 0;
        uint32_t pos = kNone;
        for (uint32_t i = lane; i < n_cls; i += 32) {
            const T y = x[i];
            if ((p == kNone || y < v || (y == v && i > p)) && (pos == kNone || y > best)) { best = y; pos = i; }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const T ob = __shfl_xor_sync(0xffffffffu, best, off);
            const uint32_t op = __shfl_xor_sync(0xffffffffu, pos, off);
            if (op != kNone && (pos == kNone || ob > best || (ob == best && op < pos))) { best = ob; pos = op; }
        }
        v = best;
        p = pos;
        if (lane == (t & 31)) { my_cls = pos; my_score = best; }
        if (((t & 31) == 31 || t + 1 == k) && lane <= (t & 31)) {
            const size_t o = row * k + (t & ~31u) + lane;
            classes[o] = my_cls;
            if (scores) scores[o] = my_score;
        }
    }
}

void launch_topk_rows(const int32_t *rows, uint32_t n_cls, uint32_t k, uint32_t *classes, int32_t *scores, size_t n, cudaStream_t st) {
    if (n) k_topk_rows<int32_t><<<(unsigned)((n + 7) / 8), 256, 0, st>>>(rows, n_cls, k, classes, scores, n);
}
void launch_topk_rows(const double *rows, uint32_t n_cls, uint32_t k, uint32_t *classes, double *scores, size_t n, cudaStream_t st) {
    if (n) k_topk_rows<double><<<(unsigned)((n + 7) / 8), 256, 0, st>>>(rows, n_cls, k, classes, scores, n);
}

void launch_relunorm_emul(const int32_t *in, uint32_t n_in, int level_shift, int8_t *out, uint32_t out_stride, size_t n, cudaStream_t st) {
    if (n) k_relunorm_emul<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(in, n_in, level_shift, out, out_stride, n);
}
void launch_expand_image(const int8_t *img, int32_t *planes, uint32_t C, uint32_t elems, size_t n, cudaStream_t st) {
    const size_t total = n * C * elems;
    if (total) k_expand_image<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(img, planes, C, elems, n);
}
void launch_conv_renorm(int32_t *planes, uint32_t elems_per_image, size_t n, cudaStream_t st) {
    if (n && elems_per_image) k_conv_renorm<<<(unsigned)n, 256, 0, st>>>(planes, elems_per_image, n);
}
void launch_i32_to_i8(const int32_t *in, uint32_t n_in, int8_t *out, uint32_t out_stride, size_t n, cudaStream_t st) {
    const size_t total = n * out_stride;
    if (total) k_i32_to_i8<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(in, n_in, out, out_stride, n);
}

// bnm_compare_engines_device off the one-pass kernel: the two engines' labels, compared and scored by a grid-stride loop whose
// warps count with EngineTally, as fc_engines_kernel's epilogue does.  The loop bound is uniform per block: every warp runs
// every ballot.
__global__ void __launch_bounds__(256) k_engine_counts(const uint32_t *__restrict__ labels_c, const uint32_t *__restrict__ labels_py,
                                                        const uint32_t *__restrict__ truth, size_t n, uint32_t n_classes,
                                                        unsigned long long *counts) {
    EngineTally tally;
    for (size_t base = (size_t)blockIdx.x * blockDim.x; base < n; base += (size_t)gridDim.x * blockDim.x) {
        const size_t i = base + threadIdx.x;
        const bool row = i < n;
        tally.add(row, row ? labels_c[i] : 0u, row ? labels_py[i] : 0u, row && truth ? truth[i] : ~0u, n_classes);
    }
    tally.flush(counts);
    if (blockIdx.x == 0 && threadIdx.x == 0) atomicAdd(&counts[0], (unsigned long long)n);
}

void launch_engine_counts(const uint32_t *labels_c, const uint32_t *labels_py, const uint32_t *truth, size_t n, uint32_t n_classes,
                          unsigned long long *counts, cudaStream_t st) {
    if (n) k_engine_counts<<<(unsigned)std::min<size_t>((n + 255) / 256, 1024), 256, 0, st>>>(labels_c, labels_py, truth, n, n_classes, counts);
}

// ------------------------------------------------------------------------------------------------
// The emulator's CNN front-end (BitNetMCU.py:435-445, 459-526) as one kernel, step for step the layered route of emulate_device
// (capi.cu): input scaling; conv1 (1 -> C), ReLU, renormalisation over the image's C*196 outputs; depthwise conv2, ReLU,
// renormalisation over C*144, 2x2 max-pool; depthwise conv3, ReLU, renormalisation over C*16, 2x2 max-pool; the (C, 2, 2)
// flatten.  Convolutions follow k_conv33relu: output (y, x) = sum of w[3 dr + dc] * in[y + dr][x + dc], no shift.
// Thread = (image, channel), ipb images per CTA.  Each renormalisation needs the maximum over all channels of the image (a
// shared-memory atomicMax, then a barrier), so conv1 and conv2 run twice: once for the maximum, once to renormalise what they
// recompute.  The one intermediate in shared memory is a channel's renormalised conv1 plane (14 rows of 16 bytes, 57 words apart:
// no bank conflicts); conv2's pooled outputs and conv3's outputs stay in registers.  conv1 and conv2 take three dp4a per output
// over 4-byte sliding windows of their input rows (the fourth weight byte is zero); conv3 is 9 IMAD per output.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kCnnEmulThreads = 256, kCnnEmulMaxImages = 16;
constexpr uint32_t kEmulImgStride = 260;     // bytes per scaled 16x16 image in shared memory (65 words)
constexpr uint32_t kEmulC1Words = 57;        // words per renormalised conv1 plane

// the 4-byte windows starting at bytes 0 .. kW-1 of a 16-byte row (four words; bytes past the row read as zero)
template <int kW>
__device__ __forceinline__ void row_windows(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, uint32_t (&win)[kW]) {
    const uint32_t w[5] = {w0, w1, w2, w3, 0u};
#pragma unroll
    for (int x = 0; x < kW; x++) win[x] = __funnelshift_r(w[x >> 2], w[(x >> 2) + 1], 8 * (x & 3));
}
__device__ __forceinline__ int pack_taps(const int8_t *k) {   // one kernel row (k[0], k[1], k[2], 0) as int8x4
    return (int)((uint32_t)(uint8_t)k[0] | (uint32_t)(uint8_t)k[1] << 8 | (uint32_t)(uint8_t)k[2] << 16);
}

// conv1 + ReLU of one channel over the scaled image im (16 rows of 16 bytes).  kRenorm false: returns the maximum.  kRenorm true:
// stores the renormalised rows into the plane c1 (14 rows x 4 words) and returns 0.
template <bool kRenorm>
__device__ __forceinline__ int emul_conv1(const uint32_t *im, const int (&k)[3], double scale, uint32_t *c1) {
    uint32_t win[3][14];
    int m = 0;
#pragma unroll
    for (int y = 0; y < 16; y++) {
        row_windows<14>(im[4 * y], im[4 * y + 1], im[4 * y + 2], im[4 * y + 3], win[y % 3]);
        if (y < 2) continue;
        const int r = y - 2;
        uint32_t out[4] = {0u, 0u, 0u, 0u};
#pragma unroll
        for (int x = 0; x < 14; x++) {
            int s = __dp4a((int)win[r % 3][x], k[0], 0);
            s = __dp4a((int)win[(r + 1) % 3][x], k[1], s);
            s = __dp4a((int)win[(r + 2) % 3][x], k[2], s);
            s = max(s, 0);
            if (kRenorm) out[x >> 2] |= (uint32_t)conv_renorm(s, scale) << (8 * (x & 3));
            else m = max(m, s);
        }
        if (kRenorm)
#pragma unroll
            for (int j = 0; j < 4; j++) c1[4 * r + j] = out[j];
    }
    return m;
}

// conv2 + ReLU of one channel over its renormalised conv1 plane c1.  kRenorm false: returns the maximum.  kRenorm true:
// renormalises, max-pools 2x2, runs conv3 (taps w3) + ReLU on the pooled rows as they complete into u and returns u's maximum.
template <bool kRenorm>
__device__ __forceinline__ int emul_conv2(const uint32_t *c1, const int (&k)[3], double scale, const int8_t *w3, int (&u)[4][4]) {
    uint32_t win[3][12];
    int even[12];   // the renormalised even row awaiting its odd partner
    int pl[3][6];   // the last three pooled rows
    int m = 0;
#pragma unroll
    for (int y = 0; y < 14; y++) {
        row_windows<12>(c1[4 * y], c1[4 * y + 1], c1[4 * y + 2], c1[4 * y + 3], win[y % 3]);
        if (y < 2) continue;
        const int r = y - 2;
#pragma unroll
        for (int x = 0; x < 12; x++) {
            int s = __dp4a((int)win[r % 3][x], k[0], 0);
            s = __dp4a((int)win[(r + 1) % 3][x], k[1], s);
            s = __dp4a((int)win[(r + 2) % 3][x], k[2], s);
            s = max(s, 0);
            if (!kRenorm) {
                m = max(m, s);
            } else if ((r & 1) == 0) {
                even[x] = conv_renorm(s, scale);
            } else {
                const int v = max(even[x], conv_renorm(s, scale));
                pl[(r >> 1) % 3][x >> 1] = (x & 1) ? max(pl[(r >> 1) % 3][x >> 1], v) : v;
            }
        }
        if (kRenorm && (r & 1) && (r >> 1) >= 2) {
            const int q = (r >> 1) - 2;   // conv3 output row
#pragma unroll
            for (int x = 0; x < 4; x++) {
                int s = 0;
#pragma unroll
                for (int dr = 0; dr < 3; dr++)
#pragma unroll
                    for (int dc = 0; dc < 3; dc++) s += (int)w3[3 * dr + dc] * pl[(q + dr) % 3][x + dc];
                u[q][x] = max(s, 0);
                m = max(m, u[q][x]);
            }
        }
    }
    return m;
}

// The front-end of a CTA's images img0 .. img0 + ipb - 1 from their scaled rows on, which the calling kernel has stored into s_img
// (shared memory after s_max: [ipb][kEmulImgStride / 4] words, bytes 4w .. 4w + 3 of a row in its word w; zeros for images past n)
// without a barrier since: the three convolutions with their renormalisations and pools, then the features.
__device__ __forceinline__ void cnn_emul_convs(uint32_t *s_emul, const int8_t *__restrict__ w1, const int8_t *__restrict__ w2,
                                               const int8_t *__restrict__ w3, uint32_t C, uint32_t ipb, int8_t *__restrict__ feats,
                                               uint32_t feat_stride, size_t n, size_t img0) {
    int *s_max = reinterpret_cast<int *>(s_emul);                  // [3][ipb]: the image maxima of conv1, conv2, conv3
    uint32_t *s_img = s_emul + 3 * ipb;                             // [ipb][kEmulImgStride / 4]
    uint32_t *s_c1 = s_img + ipb * (kEmulImgStride / 4);            // [ipb * C][kEmulC1Words]
    const uint32_t t = threadIdx.x;
    if (t < 3 * ipb) s_max[t] = 0;
    __syncthreads();

    const bool active = t < ipb * C;
    const uint32_t il = active ? t / C : 0, ch = active ? t % C : 0;
    int k1[3], k2[3];
#pragma unroll
    for (int r = 0; r < 3; r++) {
        k1[r] = pack_taps(w1 + ch * 9 + 3 * r);
        k2[r] = pack_taps(w2 + ch * 9 + 3 * r);
    }
    const uint32_t *im = s_img + il * (kEmulImgStride / 4);
    uint32_t *c1 = s_c1 + t * kEmulC1Words;
    int u[4][4];   // conv3 + ReLU

    if (active) atomicMax(&s_max[il], emul_conv1<false>(im, k1, 0.0, c1));
    __syncthreads();
    if (active) {
        emul_conv1<true>(im, k1, conv_renorm_scale(s_max[il]), c1);
        atomicMax(&s_max[ipb + il], emul_conv2<false>(c1, k2, 0.0, w3 + ch * 9, u));
    }
    __syncthreads();
    if (active) atomicMax(&s_max[2 * ipb + il], emul_conv2<true>(c1, k2, conv_renorm_scale(s_max[ipb + il]), w3 + ch * 9, u));
    __syncthreads();
    if (active && img0 + il < n) {
        const double sc = conv_renorm_scale(s_max[2 * ipb + il]);
        uint32_t f = 0;
#pragma unroll
        for (int py = 0; py < 2; py++)
#pragma unroll
            for (int px = 0; px < 2; px++) {
                const int v = max(max(conv_renorm(u[2 * py][2 * px], sc), conv_renorm(u[2 * py][2 * px + 1], sc)),
                                  max(conv_renorm(u[2 * py + 1][2 * px], sc), conv_renorm(u[2 * py + 1][2 * px + 1], sc)));
                f |= (uint32_t)v << (8 * (2 * py + px));   // flatten (C, 2, 2): feature 4 ch + 2 py + px
            }
        uint32_t *row = reinterpret_cast<uint32_t *>(feats + (img0 + il) * feat_stride);
        row[ch] = f;
        for (uint32_t w = C + ch; w < feat_stride / 4; w += C) row[w] = 0u;   // the row's zero padding
    }
}

__global__ void __launch_bounds__(kCnnEmulThreads, 2)
k_cnn_emul_frontend(const float *__restrict__ images, const int8_t *__restrict__ w1, const int8_t *__restrict__ w2,
                    const int8_t *__restrict__ w3, uint32_t C, uint32_t ipb, int8_t *__restrict__ feats, uint32_t feat_stride, size_t n) {
    extern __shared__ __align__(16) uint32_t s_emul[];
    uint32_t *s_img = s_emul + 3 * ipb;                             // [ipb][kEmulImgStride / 4]
    const uint32_t t = threadIdx.x, lane = t & 31;
    const size_t img0 = (size_t)blockIdx.x * ipb;

    // input scaling (BitNetMCU.py:435-436): warp w scales images w, w + 8, ...; lane l holds elements 4l .. 4l+3 and 128 + 4l ..
    for (uint32_t il = t >> 5; il < ipb; il += kCnnEmulThreads / 32) {
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
        if (img0 + il < n) {
            const float4 *x = reinterpret_cast<const float4 *>(images + (img0 + il) * 256);
            a = x[lane];
            b = x[lane + 32];
        }
        float m = fmax_nan(fmax_nan(fmax_nan(fabsf(a.x), fabsf(a.y)), fmax_nan(fabsf(a.z), fabsf(a.w))),
                           fmax_nan(fmax_nan(fabsf(b.x), fabsf(b.y)), fmax_nan(fabsf(b.z), fabsf(b.w))));
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) m = fmax_nan(m, __shfl_xor_sync(0xffffffffu, m, off));
        const float sc = quant_scale(m);
        auto pack = [&](float4 v) {
            return (uint32_t)(quant_pixel(v.x, sc) & 255) | (uint32_t)(quant_pixel(v.y, sc) & 255) << 8 |
                   (uint32_t)(quant_pixel(v.z, sc) & 255) << 16 | (uint32_t)(quant_pixel(v.w, sc) & 255) << 24;
        };
        s_img[il * (kEmulImgStride / 4) + lane] = pack(a);
        s_img[il * (kEmulImgStride / 4) + 32 + lane] = pack(b);
    }
    cnn_emul_convs(s_emul, w1, w2, w3, C, ipb, feats, feat_stride, n, img0);
}

// the same front-end on rows already scaled (k_quantize_windows' output): warp w copies rows w, w + 8, ... into s_img, lane l
// words l and 32 + l of its row; the scaling rule is the float kernel's, so the features are too
__global__ void __launch_bounds__(kCnnEmulThreads, 2)
k_cnn_emul_frontend_i8(const int8_t *__restrict__ images, const int8_t *__restrict__ w1, const int8_t *__restrict__ w2,
                       const int8_t *__restrict__ w3, uint32_t C, uint32_t ipb, int8_t *__restrict__ feats, uint32_t feat_stride, size_t n) {
    extern __shared__ __align__(16) uint32_t s_emul[];
    uint32_t *s_img = s_emul + 3 * ipb;                             // [ipb][kEmulImgStride / 4]
    const uint32_t t = threadIdx.x, lane = t & 31;
    const size_t img0 = (size_t)blockIdx.x * ipb;
    for (uint32_t il = t >> 5; il < ipb; il += kCnnEmulThreads / 32) {
        uint32_t a = 0u, b = 0u;
        if (img0 + il < n) {
            const uint32_t *x = reinterpret_cast<const uint32_t *>(images + (img0 + il) * 256);
            a = x[lane];
            b = x[lane + 32];
        }
        s_img[il * (kEmulImgStride / 4) + lane] = a;
        s_img[il * (kEmulImgStride / 4) + 32 + lane] = b;
    }
    cnn_emul_convs(s_emul, w1, w2, w3, C, ipb, feats, feat_stride, n, img0);
}

static uint32_t cnn_emul_ipb(uint32_t C) { return std::min(kCnnEmulMaxImages, kCnnEmulThreads / C); }

// kernel (k_cnn_emul_frontend or k_cnn_emul_frontend_i8) on n images: a CTA per ipb images
template <class In>
static bool launch_cnn_emul(void (*kernel)(const In *, const int8_t *, const int8_t *, const int8_t *, uint32_t, uint32_t, int8_t *,
                                           uint32_t, size_t),
                            const In *images, const int8_t *w1, const int8_t *w2, const int8_t *w3, uint32_t channels, int8_t *features,
                            uint32_t feat_stride, size_t n, cudaStream_t st) {
    if (channels == 0 || channels > kCnnEmulMaxChannels) return false;
    if (n == 0) return true;
    const uint32_t ipb = cnn_emul_ipb(channels);
    const size_t smem = 4 * ((size_t)3 * ipb + ipb * (kEmulImgStride / 4) + (size_t)ipb * channels * kEmulC1Words);
    if (!raise_smem_limit((const void *)kernel, smem)) return false;
    kernel<<<(unsigned)((n + ipb - 1) / ipb), kCnnEmulThreads, smem, st>>>(images, w1, w2, w3, channels, ipb, features, feat_stride, n);
    return true;
}

bool launch_cnn_emul_frontend(const float *images, const int8_t *w1, const int8_t *w2, const int8_t *w3, uint32_t channels,
                              int8_t *features, uint32_t feat_stride, size_t n, cudaStream_t st) {
    return launch_cnn_emul(k_cnn_emul_frontend, images, w1, w2, w3, channels, features, feat_stride, n, st);
}

bool launch_cnn_emul_frontend_i8(const int8_t *images, const int8_t *w1, const int8_t *w2, const int8_t *w3, uint32_t channels,
                                 int8_t *features, uint32_t feat_stride, size_t n, cudaStream_t st) {
    return launch_cnn_emul(k_cnn_emul_frontend_i8, images, w1, w2, w3, channels, features, feat_stride, n, st);
}

// ------------------------------------------------------------------------------------------------
// processconv33ReLU / processmaxpool22, one thread per output element
// ------------------------------------------------------------------------------------------------
__global__ void k_conv33relu(const int32_t *__restrict__ act, const int8_t *__restrict__ w, uint32_t n_w, uint32_t xy,
                             uint32_t n_shift, int32_t *__restrict__ out, size_t n) {
    const uint32_t oxy = xy - 2;
    size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n * oxy * oxy) return;
    size_t item = idx / (oxy * oxy);
    uint32_t r = idx % (oxy * oxy), oy = r / oxy, ox = r % oxy;
    const int32_t *p = act + item * xy * xy + oy * xy + ox;
    const int8_t *k = w + (item % n_w) * 9;
    int32_t s = 0;
#pragma unroll
    for (int dr = 0; dr < 3; dr++)
#pragma unroll
        for (int dc = 0; dc < 3; dc++) s += (int32_t)k[3 * dr + dc] * p[dr * xy + dc];
    out[idx] = s < 0 ? 0 : (s >> n_shift);   // no rounding, no clip (inference.c:261-272)
}

__global__ void k_maxpool22(const int32_t *__restrict__ act, uint32_t xy, int32_t *__restrict__ out, size_t n) {
    const uint32_t o = xy / 2;
    size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n * o * o) return;
    size_t item = idx / (o * o);
    uint32_t r = idx % (o * o), oy = r / o, ox = r % o;
    const int32_t *p = act + item * xy * xy + (2 * oy) * xy + 2 * ox;
    out[idx] = max(max(p[0], p[1]), max(p[xy], p[xy + 1]));
}

void launch_conv33relu(const int32_t *act, const int8_t *w, uint32_t n_w, uint32_t xy, uint32_t n_shift, int32_t *out, size_t n,
                       cudaStream_t st) {
    size_t total = n * (xy - 2) * (xy - 2);
    if (total == 0) return;
    k_conv33relu<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(act, w, n_w, xy, n_shift, out, n);
}
void launch_maxpool22(const int32_t *act, uint32_t xy, int32_t *out, size_t n, cudaStream_t st) {
    size_t total = n * (xy / 2) * (xy / 2);
    if (total == 0) return;
    k_maxpool22<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(act, xy, out, n);
}

// ------------------------------------------------------------------------------------------------
// Fused CNN front-end for the 16x16 geometry (BitNetMCU_MNIST_dll.c:64-80).
// thread = (image, channel).  conv1 (int8 x int8) runs on dp4a over 4-byte sliding windows that are built
// once per image in shared memory and broadcast to all channel threads; conv2 (conv1 outputs are < 2^15: int8 x int8
// x 9 >> 4 <= 9216) on dp2a over packed int16 pairs, 5 instructions per output instead of 9 IMADs; conv3
// (int32 x int8) on IMAD; rolling line buffers in registers; pools folded in; ReLUNorm over the C*4 features of
// an image via a shared-memory max.  n_shift is the literal 4 of dll.c:71-74.  Bound: the FMA pipe (IMAD/IDP issue).
// ------------------------------------------------------------------------------------------------
constexpr int kCnnThreads = 256;

__global__ void __launch_bounds__(kCnnThreads) k_cnn_frontend16(const int8_t *__restrict__ images, const int8_t *__restrict__ w1,
                                                                const int8_t *__restrict__ w2, const int8_t *__restrict__ w3,
                                                                uint32_t C, uint32_t ipb, int8_t *__restrict__ feats,
                                                                uint32_t feat_stride, size_t n) {
    extern __shared__ uint32_t s_mem[];
    uint32_t *s_img = s_mem;               // [ipb][64] words = 16 rows x 16 bytes
    uint32_t *s_win = s_mem + ipb * 64;    // [ipb][16][14] sliding 4-byte windows
    int *s_max = reinterpret_cast<int *>(s_win + ipb * 224);  // [ipb]
    const uint32_t t = threadIdx.x;
    const bool active = t < ipb * C;
    const uint32_t il = active ? t / C : 0, ch = active ? t % C : 0;

    int w1p[3], w2p[3], k3[9], w2v, w2s;   // per kernel row: (w0, w1, w2, 0) packed as int8x4
    {
        const int8_t *a = w1 + ch * 9, *b = w2 + ch * 9, *c = w3 + ch * 9;
#pragma unroll
        for (int r = 0; r < 3; r++) {
            w1p[r] = (int)((uint32_t)(uint8_t)a[3 * r] | ((uint32_t)(uint8_t)a[3 * r + 1] << 8) | ((uint32_t)(uint8_t)a[3 * r + 2] << 16));
            w2p[r] = (int)((uint32_t)(uint8_t)b[3 * r] | ((uint32_t)(uint8_t)b[3 * r + 1] << 8) | ((uint32_t)(uint8_t)b[3 * r + 2] << 16));
        }
#pragma unroll
        for (int i = 0; i < 9; i++) k3[i] = c[i];
        w2v = (int)((uint32_t)(uint8_t)b[2] | ((uint32_t)(uint8_t)b[5] << 8));   // third-column taps of rows 0 and 1
        w2s = (int)(uint32_t)(uint8_t)b[8];                                      // third-column tap of row 2
    }

    const size_t n_groups = (n + ipb - 1) / ipb;
    for (size_t g = blockIdx.x; g < n_groups; g += gridDim.x) {
        const size_t img_base = g * ipb;
        for (uint32_t idx = t; idx < ipb * 64; idx += kCnnThreads) {
            size_t img = img_base + idx / 64;
            s_img[idx] = img < n ? reinterpret_cast<const uint32_t *>(images)[img * 64 + (idx & 63)] : 0u;
        }
        if (t < ipb) s_max[t] = 0;
        __syncthreads();
        for (uint32_t idx = t; idx < ipb * 224; idx += kCnnThreads) {
            uint32_t im = idx / 224, r = (idx % 224) / 14, x = idx % 14;
            uint32_t lo = s_img[im * 64 + r * 4 + (x >> 2)];
            uint32_t hi = (x >> 2) < 3 ? s_img[im * 64 + r * 4 + (x >> 2) + 1] : 0u;
            s_win[idx] = __funnelshift_r(lo, hi, 8 * (x & 3));
        }
        __syncthreads();

        int f[4] = {0, 0, 0, 0};
        if (active) {
            const uint32_t *win = s_win + il * 224;
            uint32_t c1[3][14];   // rolling conv1 rows as int16 pairs: c1[.][x] = (v[x], v[x+1]), c1[.][13] = (v[13], 0)
            int c2e[12];     // even conv2 row awaiting its odd partner
            int pl[3][6];    // rolling pooled rows
            int c3e[4];
#pragma unroll
            for (int y = 0; y < 14; y++) {
                int v1[14];
#pragma unroll
                for (int x = 0; x < 14; x++) {
                    int s = __dp4a((int)win[(y + 0) * 14 + x], w1p[0], 0);
                    s = __dp4a((int)win[(y + 1) * 14 + x], w1p[1], s);
                    s = __dp4a((int)win[(y + 2) * 14 + x], w1p[2], s);
                    v1[x] = max(s, 0) >> 4;
                }
#pragma unroll
                for (int x = 0; x < 13; x++) c1[y % 3][x] = __byte_perm((uint32_t)v1[x], (uint32_t)v1[x + 1], 0x5410);
                c1[y % 3][13] = (uint32_t)v1[13];
                if (y >= 2) {
                    const int r = y - 2;  // conv2 output row
                    int v[12];
#pragma unroll
                    for (int x = 0; x < 12; x++) {
                        // 9 taps in 5 dp2a: columns x, x+1 of the three rows as horizontal pairs; column x+2 of rows r, r+1 as a
                        // vertical pair (one PRMT on the under-used ALU pipe); column x+2 of row r+2 alone
                        int s = __dp2a_lo((int)c1[r % 3][x], w2p[0], 0);
                        s = __dp2a_lo((int)c1[(r + 1) % 3][x], w2p[1], s);
                        s = __dp2a_lo((int)c1[(r + 2) % 3][x], w2p[2], s);
                        s = __dp2a_lo((int)__byte_perm(c1[r % 3][x + 2], c1[(r + 1) % 3][x + 2], 0x5410), w2v, s);
                        s = __dp2a_lo((int)c1[(r + 2) % 3][x + 2], w2s, s);
                        v[x] = max(s, 0) >> 4;
                    }
                    if ((r & 1) == 0) {
#pragma unroll
                        for (int x = 0; x < 12; x++) c2e[x] = v[x];
                    } else {
                        const int p = r >> 1;  // pooled row 0..5
#pragma unroll
                        for (int j = 0; j < 6; j++) pl[p % 3][j] = max(max(c2e[2 * j], c2e[2 * j + 1]), max(v[2 * j], v[2 * j + 1]));
                        if (p >= 2) {
                            const int q = p - 2;  // conv3 output row 0..3
                            int u[4];
#pragma unroll
                            for (int x = 0; x < 4; x++) {
                                int s = 0;
#pragma unroll
                                for (int dr = 0; dr < 3; dr++)
#pragma unroll
                                    for (int dc = 0; dc < 3; dc++) s += k3[3 * dr + dc] * pl[(q + dr) % 3][x + dc];
                                u[x] = max(s, 0) >> 4;
                            }
                            if ((q & 1) == 0) {
#pragma unroll
                                for (int x = 0; x < 4; x++) c3e[x] = u[x];
                            } else {
#pragma unroll
                                for (int j = 0; j < 2; j++)
                                    f[(q >> 1) * 2 + j] = max(max(c3e[2 * j], c3e[2 * j + 1]), max(u[2 * j], u[2 * j + 1]));
                            }
                        }
                    }
                }
            }
            atomicMax(&s_max[il], max(max(f[0], f[1]), max(f[2], f[3])));
        }
        __syncthreads();
        if (active && img_base + il < n) {
            // ReLUNorm over the C*4 features of this image (dll.c:80); all features are >= 0 here
            const uint32_t shift = relunorm_shift(s_max[il]);
            const int rounding = (int)((1u << shift) >> 1);
            uint32_t packed = 0;
#pragma unroll
            for (int j = 0; j < 4; j++) packed |= (uint32_t)min(127, (f[j] + rounding) >> shift) << (8 * j);
            *reinterpret_cast<uint32_t *>(feats + (img_base + il) * feat_stride + ch * 4) = packed;
        }
        __syncthreads();
    }
}

// Static range of conv3's inputs for given HOST weights (int8 [C][9] each): conv1 sums are at most 127 * (sum of positive taps) +
// 128 * (sum of |negative taps|) for int8 pixels, ReLU >> 4 of that bounds conv2's inputs (all >= 0), so only conv2's positive taps
// raise its maximum; ReLU >> 4 again bounds the pooled values.  Returns the largest bound over the channels.  (SURVEY.md
// section 7: per-channel static range proofs.)
long long cnn_conv3_bound(const int8_t *w1, const int8_t *w2, uint32_t channels) {
    long long bound = 0;
    for (uint32_t c = 0; c < channels; c++) {
        long long pos1 = 0, neg1 = 0, pos2 = 0;
        for (int k = 0; k < 9; k++) {
            const int a = w1[c * 9 + k], b = w2[c * 9 + k];
            if (a > 0) pos1 += a; else neg1 -= a;
            if (b > 0) pos2 += b;
        }
        const long long b1 = (127 * pos1 + 128 * neg1) >> 4;
        bound = std::max(bound, (b1 * pos2) >> 4);
    }
    return bound;
}

CnnFrontendKernel cnn_frontend_kernel(uint32_t channels, uint32_t xy, int frontend) {
    if (xy != 16 || channels == 0) return kCnnFrontendNone;
    if (frontend != 1 && cnn_frontend_tc_supported(channels, xy)) return kCnnFrontendTensorCores;
    return frontend == 2 || channels > kCnnThreads ? kCnnFrontendNone : kCnnFrontendCudaCores;
}

bool launch_cnn_frontend(const int8_t *images, const int8_t *w1, const int8_t *w2, const int8_t *w3, uint32_t channels,
                         uint32_t xy, int8_t *features, uint32_t feat_stride, size_t n, int sm_count, int frontend, int *d_err,
                         bool conv3_fits_u16, cudaStream_t st) {
    const CnnFrontendKernel kernel = cnn_frontend_kernel(channels, xy, frontend);
    if (kernel == kCnnFrontendNone) return false;
    if (n == 0) return true;
    if (kernel == kCnnFrontendTensorCores)
        return launch_cnn_frontend_tc(images, w1, w2, w3, channels, xy, features, feat_stride, n, sm_count, d_err, conv3_fits_u16, st);
    uint32_t ipb = kCnnThreads / channels;
    size_t smem = (size_t)ipb * (64 + 224) * 4 + ipb * 4;
    size_t n_groups = (n + ipb - 1) / ipb;
    unsigned grid = (unsigned)(n_groups < (size_t)sm_count * 2 ? n_groups : (size_t)sm_count * 2);
    k_cnn_frontend16<<<grid, kCnnThreads, smem, st>>>(images, w1, w2, w3, channels, ipb, features, feat_stride, n);
    return true;
}

}  // namespace bnm
