// cnn_wgmma.cu -- CNN front-end (BitNetMCU_MNIST_dll.c:64-80) with conv1 on the tensor cores (wgmma) and the depthwise tail on
// the CUDA cores, fed from shared memory.
//
// conv1 (processconv33ReLU #1, inference.c:238-277 called at dll.c:71) is the one convolution of the chain with a reduction to
// share: 1 input channel -> C output channels, out1[c][p] = sum_t w1[c][t] * patch[p][t].  conv2 / conv3 are depthwise
// (groups = C, models.py:111-118): as GEMMs they are block diagonal (< 2 % tensor utilisation) and stay on the CUDA cores.
//
//     D[M = (image, channel)][N = position]  =  A[(image, channel)][K = (image slot, tap)]  x  B[position][K]^T
//
//   * a TILE is 128 consecutive (image, channel) items; one warpgroup computes it as two m64 halves, in four pieces of 64
//     positions (four conv1 rows, positions laid out with a row stride of 16: N = 224 = 14 rows x 16);
//   * B is the im2col matrix of the images a tile touches: one 16-byte row (9 taps + padding) per (image, position), images side
//     by side along K (16 bytes each);
//   * A holds w1: row (image slot s, channel c) carries w1[c][0..8] in K-chunk s and zeros elsewhere, so one MMA computes conv1
//     of up to 128 / C images at once.  Tiles ignore image boundaries (item = image * C + channel), so every row is used for any
//     C that is a multiple of 16; a GROUP = 128 / gcd(C, 128) images is a whole number of tiles;
//   * both operands use the no-swizzle K-major canonical layout (8 rows x 16 bytes core matrices) with K-chunks a whole plane
//     apart: [K chunk][row][16 B], LBO = plane size, SBO = 128.
//
// The accumulators are staged in shared memory as ReLU(x) >> 4 uint16 pairs, one 14-row plane per item, so that thread r then
// runs the depthwise tail of item r alone:
//   conv2, 12 x 12 outputs x 9 taps (dll.c:72): IDP.2A over int16 pairs, 5 per output: rows are processed in pairs (y, y+1) that
//                                               share the vertical pair of their third column
//   maxpool (dll.c:73)                        : taken on the raw sums BEFORE ReLU >> 4 (both are monotone)
//   conv3 (dll.c:74), maxpool (dll.c:76)      : IMAD (int32 x int8), pooled the same way (or IDP.2A when the inputs fit 16 bits)
//   ReLUNorm over the C*4 features (dll.c:80)  : per-image maximum through shared memory once the group's tiles are done
// All integer: bit-exact with the reference.
#include <cstdio>
#include <cstdlib>

#include "kernels.h"
#include "sm90_ptx.cuh"

namespace bnm {

constexpr uint32_t kPlaneBytes = 224 * 16;   // im2col plane of one image: 14 rows x 16 positions x 16 bytes
constexpr uint32_t kStageWords = 116;        // staged conv1 plane of one item: 14 rows x 8 words, padded so that the 16-byte
                                             // row loads of eight consecutive items fall into distinct banks

struct CnnTcParams {
    const int8_t *images;
    const int8_t *w1, *w2, *w3;
    int8_t *feats;
    uint32_t feat_stride;
    size_t n;
    uint32_t C;
    uint32_t G, T;                 // images / tiles per group
    uint32_t a_plane_bytes;        // 128 rows x 16 B = 2048 (K-chunk stride of A)
    uint32_t a_phase_bytes;        // one tile phase of A: n_chunks_max * 2048
    uint32_t n_chunks_max;         // K-chunks (image slots) per tile, rounded up to even
    // shared memory carve-up (byte offsets from the 128-aligned base)
    uint32_t off_a, off_b, off_img, off_stage, off_raw, off_wc, off_imax;
    size_t n_groups;
};

__device__ __forceinline__ uint32_t pack_relu_u16(int hi, int lo) {
    uint32_t d;   // (clamp(hi, 0, 65535) << 16) | clamp(lo, 0, 65535): the ReLU comes with the conversion
    asm("cvt.pack.sat.u16.s32 %0, %1, %2;" : "=r"(d) : "r"(hi), "r"(lo));
    return d;
}

// (uint16, uint16) . (int8, int8) + c: pooled conv2 outputs reach 65535, beyond the int16 range of __dp2a_lo(int, int, int)
__device__ __forceinline__ int dp2a_u16_s8(uint32_t a, int b, int c) {
    int d;
    asm("dp2a.lo.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

// per-channel weights of the depthwise tail, 16 words
struct CnnTailW {
    int w01[3];        // conv2 kernel row r: (w[r][0], w[r][1]) as int8 pair in the low two bytes
    int wva, wvb;      // third column, vertical pairs: (w[1][2], w[2][2]) for the upper row of a pair, (w[0][2], w[1][2]) for the lower
    int wsa, wsb;      // third column, single taps: (w[0][2], 0) and (w[2][2], 0)
    int k3[9];         // conv3: scalars, or -- kConv3Packed -- k3[0..6] = the same seven pair words for conv3's kernel
};

// One tile of one thread: its item's staged conv1 plane -> 4 raw features (before ReLUNorm) of this (image, channel).
// rows: 14 rows of 8 words, word j of row y = (ReLU(conv1[y][2j]) >> 4) | (ReLU(conv1[y][2j+1]) >> 4) << 16, j < 7.
// kConv3Packed: conv3's inputs (pooled conv2 outputs) are known to fit 16 bits for this model's weights (static bound, checked on
// the host), so conv3 runs on IDP.2A like conv2; otherwise int32 x int8 IMADs.
template <bool kConv3Packed>
__device__ __forceinline__ void cnn_tile_tail(const uint32_t *rows, const CnnTailW &W, int (&f)[4]) {
    uint32_t E[14][7], O[14][7];   // conv1 rows as int16 pairs: E[y][j] = (v[2j], v[2j+1]), O[y][j] = (v[2j+1], v[2j+2]); 4 rows live
    int pl[6][6];                  // pooled conv2 rows (3 live)
    int c3e[4];
    uint32_t PE[6][3], PO[6][3];   // kConv3Packed: pooled rows as uint16 pairs
#pragma unroll
    for (int y = 0; y < 14; y++) {
        {   // conv1 row y as uint16 pairs (ReLU >> 4 was applied when the accumulators were staged)
            const uint4 a = *reinterpret_cast<const uint4 *>(rows + 8 * y), b = *reinterpret_cast<const uint4 *>(rows + 8 * y + 4);
            E[y][0] = a.x; E[y][1] = a.y; E[y][2] = a.z; E[y][3] = a.w; E[y][4] = b.x; E[y][5] = b.y; E[y][6] = b.z;
#pragma unroll
            for (int j = 0; j < 6; j++) O[y][j] = __byte_perm(E[y][j], E[y][j + 1], 0x5432);
            O[y][6] = E[y][6] >> 16;
        }
        if (y >= 3 && (y & 1)) {
            // conv2 output rows (y-3, y-2) from conv1 rows R0..R3 = y-3..y, pooled into row p
            const int p = (y - 3) >> 1, R0 = y - 3, R1 = y - 2, R2 = y - 1, R3 = y;
#define BNM_P(r, x) (((x) & 1) ? O[r][(x) >> 1] : E[r][(x) >> 1])
#pragma unroll
            for (int j = 0; j < 6; j++) {
                int a[2], b[2];
#pragma unroll
                for (int e = 0; e < 2; e++) {
                    const int x = 2 * j + e;
                    const int v = (int)__byte_perm(BNM_P(R1, x + 2), BNM_P(R2, x + 2), 0x5410);   // (R1[x+2], R2[x+2])
                    int s = __dp2a_lo((int)BNM_P(R0, x), W.w01[0], 0);
                    s = __dp2a_lo((int)BNM_P(R1, x), W.w01[1], s);
                    s = __dp2a_lo((int)BNM_P(R2, x), W.w01[2], s);
                    s = __dp2a_lo(v, W.wva, s);
                    a[e] = __dp2a_lo((int)BNM_P(R0, x + 2), W.wsa, s);
                    int u = __dp2a_lo((int)BNM_P(R1, x), W.w01[0], 0);
                    u = __dp2a_lo((int)BNM_P(R2, x), W.w01[1], u);
                    u = __dp2a_lo((int)BNM_P(R3, x), W.w01[2], u);
                    u = __dp2a_lo(v, W.wvb, u);
                    b[e] = __dp2a_lo((int)BNM_P(R3, x + 2), W.wsb, u);
                }
                pl[p][j] = max(__vimax3_s32_relu(a[0], a[1], b[0]), b[1]) >> 4;   // maxpool, then ReLU >> 4 (monotone: same result)
            }
#undef BNM_P
            if (!kConv3Packed) {
                if (p >= 2) {
                    const int q = p - 2;   // conv3 output row
                    int u[4];
#pragma unroll
                    for (int x = 0; x < 4; x++) {
                        int s = 0;
#pragma unroll
                        for (int dr = 0; dr < 3; dr++)
#pragma unroll
                            for (int dc = 0; dc < 3; dc++) s += W.k3[3 * dr + dc] * pl[q + dr][x + dc];
                        u[x] = s;
                    }
                    if ((q & 1) == 0) {
#pragma unroll
                        for (int x = 0; x < 4; x++) c3e[x] = u[x];
                    } else {
#pragma unroll
                        for (int j = 0; j < 2; j++)
                            f[(q >> 1) * 2 + j] = max(__vimax3_s32_relu(c3e[2 * j], c3e[2 * j + 1], u[2 * j]), u[2 * j + 1]) >> 4;
                    }
                }
            } else {
                // pooled row p as uint16 pairs, then conv3 exactly like conv2: output rows (0,1) after pooled row 3, (2,3) after row 5
#pragma unroll
                for (int j = 0; j < 3; j++) PE[p][j] = __byte_perm((uint32_t)pl[p][2 * j], (uint32_t)pl[p][2 * j + 1], 0x5410);
#pragma unroll
                for (int j = 0; j < 2; j++) PO[p][j] = __byte_perm((uint32_t)pl[p][2 * j + 1], (uint32_t)pl[p][2 * j + 2], 0x5410);
                PO[p][2] = (uint32_t)pl[p][5];
                if (p == 3 || p == 5) {
                    const int Q0 = p - 3, Q1 = p - 2, Q2 = p - 1, Q3 = p;
#define BNM_Q(r, x) (((x) & 1) ? PO[r][(x) >> 1] : PE[r][(x) >> 1])
#pragma unroll
                    for (int j = 0; j < 2; j++) {
                        int a[2], b[2];
#pragma unroll
                        for (int e = 0; e < 2; e++) {
                            const int x = 2 * j + e;
                            const int v = (int)__byte_perm(BNM_Q(Q1, x + 2), BNM_Q(Q2, x + 2), 0x5410);
                            int s = dp2a_u16_s8(BNM_Q(Q0, x), W.k3[0], 0);
                            s = dp2a_u16_s8(BNM_Q(Q1, x), W.k3[1], s);
                            s = dp2a_u16_s8(BNM_Q(Q2, x), W.k3[2], s);
                            s = dp2a_u16_s8((uint32_t)v, W.k3[3], s);
                            a[e] = dp2a_u16_s8(BNM_Q(Q0, x + 2), W.k3[5], s);
                            int u = dp2a_u16_s8(BNM_Q(Q1, x), W.k3[0], 0);
                            u = dp2a_u16_s8(BNM_Q(Q2, x), W.k3[1], u);
                            u = dp2a_u16_s8(BNM_Q(Q3, x), W.k3[2], u);
                            u = dp2a_u16_s8((uint32_t)v, W.k3[4], u);
                            b[e] = dp2a_u16_s8(BNM_Q(Q3, x + 2), W.k3[6], u);
                        }
                        f[(p == 5 ? 2 : 0) + j] = max(__vimax3_s32_relu(a[0], a[1], b[0]), b[1]) >> 4;
                    }
#undef BNM_Q
                }
            }
        }
    }
}

template <bool kConv3Packed>
__global__ void __launch_bounds__(128) k_cnn_frontend16_tc(const __grid_constant__ CnnTcParams P) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t t = threadIdx.x, lane = t & 31, warp = t >> 5;
    uint8_t *base = smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u);
    const uint32_t C = P.C, G = P.G, T = P.T;

    // ---- one-time setup: the A operand (w1 per tile phase), per-channel tail weights
    {
        uint4 *a4 = reinterpret_cast<uint4 *>(base + P.off_a);
        const uint32_t total = T * P.n_chunks_max * 128;   // 16-byte rows
        for (uint32_t i = t; i < total; i += 128) {
            const uint32_t phase = i / (P.n_chunks_max * 128), rem = i % (P.n_chunks_max * 128), chunk = rem >> 7, r = rem & 127;
            const uint32_t item = phase * 128 + r, il = item / C, ch = item % C, i0 = (phase * 128) / C;
            uint32_t q[4] = {0, 0, 0, 0};
            if (il - i0 == chunk) {
                const int8_t *w = P.w1 + ch * 9;
#pragma unroll
                for (int k = 0; k < 9; k++) q[k >> 2] |= (uint32_t)(uint8_t)w[k] << (8 * (k & 3));
            }
            a4[i] = make_uint4(q[0], q[1], q[2], q[3]);   // [phase][chunk][row][16 B]
        }
        int *wc = reinterpret_cast<int *>(base + P.off_wc);
        for (uint32_t ch = t; ch < C; ch += 128) {
            const int8_t *b = P.w2 + ch * 9, *c = P.w3 + ch * 9;
            auto pair = [](int8_t lo, int8_t hi) { return (int)((uint32_t)(uint8_t)lo | ((uint32_t)(uint8_t)hi << 8)); };
            int *o = wc + ch * 16;
            o[0] = pair(b[0], b[1]); o[1] = pair(b[3], b[4]); o[2] = pair(b[6], b[7]);
            o[3] = pair(b[5], b[8]); o[4] = pair(b[2], b[5]);
            o[5] = pair(b[2], 0); o[6] = pair(b[8], 0);
            if (kConv3Packed) {
                o[7] = pair(c[0], c[1]); o[8] = pair(c[3], c[4]); o[9] = pair(c[6], c[7]);
                o[10] = pair(c[5], c[8]); o[11] = pair(c[2], c[5]);
                o[12] = pair(c[2], 0); o[13] = pair(c[8], 0);
                o[14] = o[15] = 0;
            } else {
#pragma unroll
                for (int k = 0; k < 9; k++) o[7 + k] = c[k];
            }
        }
    }
    fence_proxy_async_smem();   // the tensor cores (async proxy) read A
    __syncthreads();

    const uint32_t a_base = smem_u32(base + P.off_a), b_base = smem_u32(base + P.off_b);
    uint32_t *s_img = reinterpret_cast<uint32_t *>(base + P.off_img);
    uint32_t *stage = reinterpret_cast<uint32_t *>(base + P.off_stage);
    int4 *raw = reinterpret_cast<int4 *>(base + P.off_raw);
    int *imax = reinterpret_cast<int *>(base + P.off_imax);
    const int *wc = reinterpret_cast<const int *>(base + P.off_wc);
    CnnTailW W;
    auto load_weights = [&](uint32_t ch) {
        const int4 *w4 = reinterpret_cast<const int4 *>(wc + ch * 16);
        const int4 q0 = w4[0], q1 = w4[1], q2 = w4[2], q3 = w4[3];
        W.w01[0] = q0.x; W.w01[1] = q0.y; W.w01[2] = q0.z; W.wva = q0.w;
        W.wvb = q1.x; W.wsa = q1.y; W.wsb = q1.z; W.k3[0] = q1.w;
        W.k3[1] = q2.x; W.k3[2] = q2.y; W.k3[3] = q2.z; W.k3[4] = q2.w;
        W.k3[5] = q3.x; W.k3[6] = q3.y; W.k3[7] = q3.z; W.k3[8] = q3.w;
    };

    for (size_t j = blockIdx.x; j < P.n_groups; j += gridDim.x) {
        if (t < 8) imax[t] = 0;
        for (uint32_t tau = 0; tau < T; tau++) {
            // ---- the tile's images -> shared memory -> im2col planes
            const uint32_t i0 = (tau * 128) / C, count = (tau * 128 + 127) / C - i0 + 1;
            const size_t first = j * G + i0;
            for (uint32_t idx = t; idx < count * 16; idx += 128)
                reinterpret_cast<uint4 *>(s_img)[idx] = first + idx / 16 < P.n ? reinterpret_cast<const uint4 *>(P.images)[first * 16 + idx]
                                                                                : make_uint4(0, 0, 0, 0);
            __syncthreads();
            // one task = four consecutive positions (y, 4 xg .. 4 xg + 3) of one image: six shared-memory words (two per image row)
            // feed four 16-byte im2col rows; 56 tasks per image (14 rows x 4 column groups, the last group holds x = 12, 13 only)
            for (uint32_t task = t; task < count * 56; task += 128) {
                const uint32_t im = task / 56, rem = task - im * 56, y = rem >> 2, xg = rem & 3;
                const uint32_t *row = s_img + im * 64 + y * 4 + xg;
                const uint32_t a0 = row[0], a1 = row[1], b0 = row[4], b1 = row[5], c0 = row[8], c1 = row[9];
                uint8_t *dst = base + P.off_b + im * kPlaneBytes + (y * 16 + xg * 4) * 16;
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    if (i < 2 || xg < 3) {
                        const uint32_t wa = i ? __funnelshift_r(a0, a1, 8 * i) : a0, wb = i ? __funnelshift_r(b0, b1, 8 * i) : b0,
                                       wcc = i ? __funnelshift_r(c0, c1, 8 * i) : c0;
                        // taps in the order of w1[c][0..8]: (a0 a1 a2 b0 | b1 b2 c0 c1 | c2 . . . | . . . .); bytes 9..15 meet zeros in A
                        uint4 q;
                        q.x = __byte_perm(wa, wb, 0x4210);
                        q.y = __byte_perm(wb, wcc, 0x5421);
                        q.z = wcc >> 16;
                        q.w = 0;
                        *reinterpret_cast<uint4 *>(dst + 16 * i) = q;
                    }
                }
            }
            fence_proxy_async_smem();   // the MMAs (async proxy) read what these generic-proxy stores wrote
            __syncthreads();
            // ---- conv1: piece k = conv1 rows 4k .. 4k+3 (im2col rows 64k .. 64k+63; the last piece runs 32 rows past the plane into
            // rows nobody reads), both 64-item halves, then staged as ReLU >> 4 uint16 pairs
            const uint32_t n_k = (count + 1) / 2;   // K-steps of 32 bytes = two image slots
#pragma unroll 1
            for (uint32_t k = 0; k < 4; k++) {
                uint32_t acc[2][32];
                wgmma_fence();
#pragma unroll 1
                for (uint32_t s = 0; s < n_k; s++) {
                    const uint64_t bd = make_smem_desc(b_base + s * 2 * kPlaneBytes + k * 64 * 16, kPlaneBytes, 128, GMMA_LAYOUT_NONE);
#pragma unroll
                    for (int hh = 0; hh < 2; hh++) {
                        const uint64_t ad = make_smem_desc(a_base + tau * P.a_phase_bytes + s * 2 * P.a_plane_bytes + hh * 64 * 16,
                                                           P.a_plane_bytes, 128, GMMA_LAYOUT_NONE);
                        wgmma_ss_n64(acc[hh], ad, bd, s != 0);
                    }
                }
                wgmma_commit();
                wgmma_wait<0>();
#pragma unroll
                for (int hh = 0; hh < 2; hh++)
#pragma unroll
                    for (int g = 0; g < 8; g++)
#pragma unroll
                        for (int r = 0; r < 2; r++) {
                            const uint32_t item = hh * 64 + warp * 16 + (lane >> 2) + 8 * r, y = 4 * k + g / 2;
                            const uint32_t word = 4 * (g & 1) + (lane & 3);   // positions 2 word, 2 word + 1 of row y
                            if (y < 14)
                                stage[item * kStageWords + 8 * y + word] = pack_relu_u16((int)acc[hh][4 * g + 2 * r + 1] >> 4, (int)acc[hh][4 * g + 2 * r] >> 4);
                        }
            }
            __syncthreads();
            // ---- depthwise tail of item r
            {
                const uint32_t item = tau * 128 + t;
                load_weights(item % C);
                int f[4] = {0, 0, 0, 0};
                cnn_tile_tail<kConv3Packed>(stage + t * kStageWords, W, f);
                raw[item] = make_int4(f[0], f[1], f[2], f[3]);
                atomicMax(&imax[item / C], max(max(f[0], f[1]), max(f[2], f[3])));
            }
            __syncthreads();   // the staging plane and the im2col buffer are reused by the next tile
        }
        // ---- ReLUNorm over the C*4 features of each image (dll.c:80): the maximum over ALL channels of the image
        for (uint32_t it = 0; it < T; it++) {
            const uint32_t item = it * 128 + t, il = item / C, ch = item - il * C;
            const size_t img = j * G + il;
            const int m = imax[il];
            const uint32_t shift = 32u - (uint32_t)__clz(m >> 7);   // bit length of max >> 7 (inference.c:41-47); features are >= 0
            const int rounding = (int)((1u << shift) >> 1);
            const int4 v = raw[item];
            const uint32_t packed = (uint32_t)min(127, (v.x + rounding) >> shift) | ((uint32_t)min(127, (v.y + rounding) >> shift) << 8) |
                                    ((uint32_t)min(127, (v.z + rounding) >> shift) << 16) | ((uint32_t)min(127, (v.w + rounding) >> shift) << 24);
            if (img < P.n) *reinterpret_cast<uint32_t *>(P.feats + img * P.feat_stride + ch * 4) = packed;
        }
        __syncthreads();   // raw / imax are reused by the next group
    }
}

static uint32_t gcd_u32(uint32_t a, uint32_t b) { return b ? gcd_u32(b, a % b) : a; }

// geometry + shared-memory carve-up for a channel count; returns the dynamic shared memory needed, 0 when the shape is not covered
static size_t cnn_tc_plan(uint32_t channels, uint32_t xy, CnnTcParams &p) {
    if (xy != 16 || channels < 16 || channels > 128 || channels % 16) return 0;
    p.C = channels;
    p.G = 128 / gcd_u32(channels, 128);
    p.T = p.G * channels / 128;
    uint32_t max_imgs = 1;
    for (uint32_t tau = 0; tau < p.T; tau++) max_imgs = std::max(max_imgs, (tau * 128 + 127) / channels - (tau * 128) / channels + 1);
    p.n_chunks_max = (max_imgs + 1) / 2 * 2;
    p.a_plane_bytes = 128 * 16;
    p.a_phase_bytes = p.n_chunks_max * p.a_plane_bytes;
    uint32_t off = 0;
    auto take = [&](uint32_t bytes) { uint32_t o = off; off += (bytes + 127) / 128 * 128; return o; };
    p.off_a = take(p.T * p.a_phase_bytes);
    // one tile's images + one spare plane (an odd image count reads one zero-weighted chunk past the last image) + 32 rows (the
    // last accumulator piece of a tile covers im2col rows 192..255 of a 224-row plane)
    p.off_b = take((max_imgs + 1) * kPlaneBytes + 32 * 16);
    p.off_img = take(max_imgs * 256);
    p.off_stage = take(128 * kStageWords * 4);
    p.off_raw = take(p.T * 128 * 16);
    p.off_wc = take(channels * 64);
    p.off_imax = take(8 * 4);
    return (size_t)off + 128;
}

bool cnn_frontend_tc_supported(uint32_t channels, uint32_t xy) {
    CnnTcParams p{};
    return cnn_tc_plan(channels, xy, p) != 0;
}

// returns false when the shape is not covered (the caller then uses k_cnn_frontend16)
bool launch_cnn_frontend_tc(const int8_t *images, const int8_t *w1, const int8_t *w2, const int8_t *w3, uint32_t channels,
                            uint32_t xy, int8_t *features, uint32_t feat_stride, size_t n, int sm_count, int *d_err,
                            bool conv3_fits_u16, cudaStream_t st) {
    (void)d_err;   // no bounded waits in this kernel
    CnnTcParams p{};
    const size_t smem = cnn_tc_plan(channels, xy, p);
    if (!smem) return false;
    p.images = images; p.w1 = w1; p.w2 = w2; p.w3 = w3; p.feats = features; p.feat_stride = feat_stride; p.n = n;
    p.n_groups = (n + p.G - 1) / p.G;
    static size_t granted = 0;
    if (smem > granted) {
        if (cudaFuncSetAttribute(k_cnn_frontend16_tc<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess ||
            cudaFuncSetAttribute(k_cnn_frontend16_tc<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
            cudaGetLastError();   // not sticky: leave no stale error behind for the caller's launch check
            return false;
        }
        granted = smem;
    }
    // as many resident CTAs as shared memory allows, persistent over the groups
    const size_t per_sm = std::max<size_t>(1, (227 * 1024) / (smem + 1024));
    const unsigned grid = (unsigned)std::min<size_t>(p.n_groups, (size_t)sm_count * per_sm);
    if (conv3_fits_u16) k_cnn_frontend16_tc<true><<<grid, 128, smem, st>>>(p);
    else k_cnn_frontend16_tc<false><<<grid, 128, smem, st>>>(p);
    return true;
}

}  // namespace bnm
