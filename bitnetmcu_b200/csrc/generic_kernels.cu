// generic_kernels.cu -- CUDA-core kernels of the engine (any layer shape):
//   * weight pre-decode  : packed exportquant words -> dense int8 planes          (reference decode rules inference.c:96-201)
//   * processfclayer     : dp4a over the decoded planes, thread-per-image tile    (inference.c:88-208)
//   * ReLUNorm           : warp-per-row, shuffle max/argmax reduction             (inference.c:23-72)
//   * processconv33ReLU / processmaxpool22 batched                                (inference.c:238-277, 300-322)
//   * fused CNN front-end: conv,conv,pool,conv,pool per channel + ReLUNorm        (BitNetMCU_MNIST_dll.c:64-80)
// These are the layer-by-layer path (BNM_PATH_LAYERS) and the front half of every CNN model; the fused
// wgmma FC chain lives in fc_wgmma.cu.
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
// ------------------------------------------------------------------------------------------------
template <bool HAS_B>
__global__ void __launch_bounds__(128) k_fc_dp4a(const int8_t *__restrict__ act, uint32_t act_stride, uint32_t act_valid,
                                                  const int4 *__restrict__ qa, const int4 *__restrict__ qb, uint32_t k4n,
                                                  uint32_t n_out, uint32_t n_pad, int32_t *__restrict__ out, size_t n) {
    extern __shared__ uint32_t s_act[];  // [128][k4n + 1]
    const uint32_t tid = threadIdx.x;
    const size_t img0 = (size_t)blockIdx.x * 128;
    const uint32_t stride = k4n + 1;
    for (uint32_t idx = tid; idx < 128 * k4n; idx += 128) {
        uint32_t im = idx / k4n, k4 = idx % k4n;
        uint32_t v = 0;
        if (img0 + im < n && k4 * 4 < act_valid) v = *reinterpret_cast<const uint32_t *>(act + (img0 + im) * act_stride + k4 * 4);
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
    static size_t granted[2] = {48 * 1024, 48 * 1024};   // opt-in dynamic shared memory granted so far, per instantiation
    const int vi = L.dense_b ? 1 : 0;
    if (smem > granted[vi]) {
        const cudaError_t e = vi ? cudaFuncSetAttribute(k_fc_dp4a<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                                 : cudaFuncSetAttribute(k_fc_dp4a<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) { cudaGetLastError(); return false; }
        granted[vi] = smem;
    }
    if (vi) k_fc_dp4a<true><<<grid, 128, smem, st>>>(act, act_stride, valid, L.quad_a, L.quad_b, k4n, L.n_out, L.n_pad, out, n);
    else k_fc_dp4a<false><<<grid, 128, smem, st>>>(act, act_stride, valid, L.quad_a, L.quad_a, k4n, L.n_out, L.n_pad, out, n);
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
// is bit-identical to the NumPy expression.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_quantize_images(const float *__restrict__ in, uint32_t elems, int8_t *__restrict__ out, size_t n) {
    const uint32_t lane = threadIdx.x & 31;
    const size_t img = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (img >= n) return;
    const float *x = in + img * elems;
    float m = 0.0f;
    for (uint32_t i = lane; i < elems; i += 32) m = fmaxf(m, fabsf(x[i]));
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
    const float scale = __fdiv_rn(127.0f, fmaxf(m, 1e-5f));
    int8_t *q = out + img * elems;
    for (uint32_t i = lane; i < elems; i += 32) {
        float y = rintf(__fmul_rn(x[i], scale));            // np.round: round half to even
        y = fminf(fmaxf(y, -128.0f), 127.0f);               // .clip(-128, 127)
        q[i] = (int8_t)(int)y;
    }
}

void launch_quantize_images(const float *in, uint32_t elems, int8_t *out, size_t n, cudaStream_t st) {
    if (n == 0 || elems == 0) return;
    k_quantize_images<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(in, elems, out, n);
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
    if (m <= 0) return;   // all-zero conv output: NumPy divides by zero here (nan); defined as zeros
    const double scale = 127.0 / (double)m;
    for (uint32_t i = threadIdx.x; i < elems; i += 256) {
        const double y = rint(__dmul_rn((double)p[i], scale));
        p[i] = (int)fmin(fmax(y, 0.0), 127.0);
    }
}

__global__ void k_i32_to_i8(const int32_t *__restrict__ in, uint32_t n_in, int8_t *__restrict__ out, uint32_t out_stride, size_t n) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n * out_stride) return;
    const size_t row = idx / out_stride;
    const uint32_t c = idx % out_stride;
    out[idx] = c < n_in ? (int8_t)in[row * n_in + c] : (int8_t)0;
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
// raise its maximum; ReLU >> 4 again bounds the pooled values.  (SURVEY.md section 7: per-channel static range proofs.)
bool cnn_conv3_fits_u16(const int8_t *w1, const int8_t *w2, uint32_t channels) {
    for (uint32_t c = 0; c < channels; c++) {
        long long pos1 = 0, neg1 = 0, pos2 = 0;
        for (int k = 0; k < 9; k++) {
            const int a = w1[c * 9 + k], b = w2[c * 9 + k];
            if (a > 0) pos1 += a; else neg1 -= a;
            if (b > 0) pos2 += b;
        }
        const long long b1 = (127 * pos1 + 128 * neg1) >> 4;
        if (((b1 * pos2) >> 4) > 65535) return false;
    }
    return true;
}

bool launch_cnn_frontend(const int8_t *images, const int8_t *w1, const int8_t *w2, const int8_t *w3, uint32_t channels,
                         uint32_t xy, int8_t *features, uint32_t feat_stride, size_t n, int sm_count, int frontend, int *d_err,
                         bool conv3_fits_u16, cudaStream_t st) {
    if (xy != 16 || channels == 0) return false;
    if (n == 0) return true;
    if (frontend != 1 && launch_cnn_frontend_tc(images, w1, w2, w3, channels, xy, features, feat_stride, n, sm_count, d_err, conv3_fits_u16, st)) return true;
    if (frontend == 2 || channels > kCnnThreads) return false;
    uint32_t ipb = kCnnThreads / channels;
    size_t smem = (size_t)ipb * (64 + 224) * 4 + ipb * 4;
    size_t n_groups = (n + ipb - 1) / ipb;
    unsigned grid = (unsigned)(n_groups < (size_t)sm_count * 2 ? n_groups : (size_t)sm_count * 2);
    k_cnn_frontend16<<<grid, kCnnThreads, smem, st>>>(images, w1, w2, w3, channels, ipb, features, feat_stride, n);
    return true;
}

}  // namespace bnm
