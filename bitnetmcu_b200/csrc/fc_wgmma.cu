// fc_wgmma.cu -- the hot path: the whole processfclayer -> ReLUNorm chain of BitMnistInference
// (BitNetMCU_MNIST_dll.c:95-121, kernels inference.c:88-208 + 23-72) as ONE persistent sm_90a kernel.  Per 128-image tile:
//
//   TMA (cp.async.bulk.tensor, SWIZZLE_128B, evict-first)  images  HBM -> smem ring
//   layer 1   wgmma s8 (SS)  A = smem image tile (64 rows per warpgroup), B = decoded int8 weights (smem) -> int32 in registers
//   ReLUNorm  on the accumulator registers: row max over the four threads that share a row (two shuffles) -> shift ->
//             clamp(x+r,0,cap)>>shift -> int8x4 pack, straight into the register fragment of the next layer's A operand
//   layer l>1 wgmma s8 (RS)  A = those registers, B = smem weights                                    -> int32 in registers
//   last      int32 logits: first-maximum argmax over the quad + 64-bit stores straight to HBM
//
// The accumulator fragment of a thread holds columns {2c, 2c+1, 8+2c, 9+2c} of every 16-column block (c = lane % 4), while the
// A fragment wants K positions {4c .. 4c+3}: instead of shuffling activations, the K axis of every hidden layer's weights is
// permuted once at model build (k_build_b_image) so that K position 4c + e of a block multiplies neuron 2c + (e & 1) + 8 (e >> 1).
// Activations never leave the registers between layers.
//
// A CTA runs one or two "pipes": each pipe has its own ring of image stages and two consumer warpgroups that take the upper and
// lower 64 rows of every tile of the pipe.  Several warpgroups keep the tensor cores busy while the others run the integer ALU
// work of ReLUNorm, which bounds this kernel.  Weights of every encoding are pre-decoded once per model into int8 planes
// (kernels.h FcLayerDev); FP130's +128 does not fit s8 and is carried by a second residual plane accumulated into the same D.
// All arithmetic is integer: results are bit-exact with the reference.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "kernels.h"
#include "sm90_ptx.cuh"

namespace bnm {

constexpr int kMaxStages = 8;              // ring stages over all pipes of a CTA
constexpr uint32_t kEmptyArrivals = 8;     // a stage is free once the 8 warps of its two consumer warpgroups are past layer 1
constexpr uint32_t kFloatQuantWarps = 8;   // float-input path: quantiser warps per CTA (one pipe next to them)
constexpr uint32_t kFloatRowsPerWarp = 128 / kFloatQuantWarps;   // rows of every tile per quantiser warp
constexpr uint32_t kFloatGroupRows = 4;    // rows per bulk copy of a quantiser warp (4 kB for 256-element rows) = rows per pass

struct ChainParams {
    int n_layers;
    uint32_t n_pad[kMaxFcLayers];     // wgmma N of layer l (multiple of 16)
    uint32_t k_steps[kMaxFcLayers];   // K/32 MMA steps per plane
    uint32_t planes[kMaxFcLayers];    // 1, or 2 when the residual plane exists
    uint32_t b_off[kMaxFcLayers];     // smem byte offset (from weight base) of the layer's first [n_pad x 32B] tile
    uint32_t in_atoms;                // layer-1 A: 128-byte SW128 atoms per row (TMA boxes per tile)
    uint32_t stage_bytes;             // in_atoms * 128 rows * 128 B
    uint32_t n_stages;                // stages per pipe
    uint32_t w_bytes;                 // weight image bytes (multiple of 16), including the zero tile
    uint32_t zero_off;                // offset of a [kN x 32 B] all-zero tile at the end of the weight image
    uint32_t off_w;                   // smem offset (from the 1024-aligned base) of the weight image
    uint32_t n_classes;
    uint32_t n_tiles;
    const uint8_t *w_image;
    int32_t *logits;
    uint32_t *labels;
    size_t n;
    int *err;
    uint32_t wait_prior_grid;         // programmatic dependent launch: read inputs only after the previous kernel has completed
    uint32_t early_trigger;           // let the next launch's CTAs take over SMs as this launch's CTAs leave (full grids only)
    // result exchange fused into the epilogue: besides logits / labels, row i of this launch is also stored at row row0 + i of
    // every destination buffer -- peer GPUs' memory mapped through CUDA IPC / P2P, written over NVLink
    uint32_t n_lab_dst, n_log_dst;
    uint32_t *lab_dst[kMaxGatherDst];
    int32_t *log_dst[kMaxGatherDst];
    size_t row0;
    uint32_t lab_u8;                  // gather launches: lab_dst are uint8 buffers (one byte per label)
    const float *fimages;             // float-input launches: float32 [n][in_elems] instead of the int8 tensor map
    uint32_t in_elems;                // real elements per image row (<= 256 for the float path)
    uint32_t off_fring;               // float-input launches: smem offset of the quantiser warps' float rings (8 warps x 2 slots x 4 kB)
};

struct FcChainPlan {
    ChainParams p{};
    uint8_t *d_w_image = nullptr;
    int *d_err = nullptr;             // error word of the bounded device-side waits: mapped pinned host memory, readable after a trap
    int *h_err = nullptr;
    size_t smem_bytes = 0;
    uint32_t in_bytes = 0;
    uint32_t max_n = 0;               // accumulator width the kernel is instantiated for: 64, 128, 192 or 256 columns
    uint32_t pipes = 1;
    int sm_count = 0;
    int device = 0;
    int overlap = 0;                  // BNM_OPT_LAUNCH_OVERLAP: 0 plain launch, 1 dependent launch + wait, 2 independent launches
    // float-input launches: one pipe, fewer int8 stages, the freed shared memory holds the quantiser warps' float rings
    uint32_t f_n_stages = 0, f_off_w = 0, f_off_fring = 0;
    size_t f_smem_bytes = 0;
    struct TmapSlot { const void *ptr = nullptr; size_t n = 0; CUtensorMap map; };
    TmapSlot tmaps[4];                // tensor maps of the most recent (pointer, n) pairs: double/triple-buffered callers hit every time
    unsigned tmap_next = 0;
    // mode 2 bookkeeping: the buffers of the previous launch on this plan (the promise "consecutive launches are independent" is
    // checked as far as the library can see it: a launch that reuses a buffer of the one before keeps the grid-dependency wait)
    const void *prev_in = nullptr, *prev_logits = nullptr, *prev_labels = nullptr;
    cudaStream_t prev_stream = nullptr;
    bool prev_valid = false;
};

// ---------------------------------------------------------------------------------------------------
// weight image: every MMA K-step reads one [n_pad x 32 B] tile in the no-swizzle K-major canonical layout
// (8-row x 16-byte core matrices; LBO = 128 B between the two K halves, SBO = 256 B between 8-row groups).
// permute_k (hidden layers, whose A comes from accumulator registers): K position p of every 16-block holds the weight of input
// neuron 2 ((p & 15) >> 2) + (p & 1) + 8 ((p >> 1) & 1) of that block.
// ---------------------------------------------------------------------------------------------------
__global__ void k_build_b_image(const int8_t *__restrict__ dense, uint32_t k_pad_src, uint32_t n_pad, uint32_t k_steps,
                                uint32_t permute_k, uint8_t *__restrict__ image) {
    size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t total = (size_t)n_pad * k_steps * 32;
    if (idx >= total) return;
    uint32_t n = idx / (k_steps * 32), k = idx % (k_steps * 32);
    const uint32_t src = permute_k ? (k & ~15u) | (2 * ((k & 15) >> 2) + (k & 1) + 8 * ((k >> 1) & 1)) : k;
    uint8_t v = src < k_pad_src ? (uint8_t)dense[(size_t)n * k_pad_src + src] : 0;
    uint32_t kb = k & 31;
    size_t off = (size_t)(k >> 5) * n_pad * 32 + (n >> 3) * 256 + (kb >> 4) * 128 + (n & 7) * 16 + (kb & 15);
    image[off] = v;
}

// ---------------------------------------------------------------------------------------------------
// ReLUNorm pieces (inference.c:23-72)
// ---------------------------------------------------------------------------------------------------
struct NormCoef { int rounding, cap; uint32_t mult; };

__device__ __forceinline__ NormCoef norm_coef(int row_max_relu) {
    // shift = bit length of (max >> 7) (inference.c:41-47).  row_max_relu = max(row max, 0): a negative row
    // maximum zeroes every output whatever the shift, so taking the maximum over relu'd values is equivalent.
    const uint32_t shift = 32u - (uint32_t)__clz(row_max_relu >> 7);
    NormCoef c;
    c.rounding = (int)((1u << shift) >> 1);                 // inference.c:51
    c.cap = (int)((128u << shift) - 1u);                    // (cap >> shift) == 127: the clip of inference.c:60-64
    c.mult = 1u << (24u - shift);                           // u * mult puts (u >> shift) into byte 3
    return c;
}
// four int32 accumulators -> four int8 (0..127) packed little-endian.  1 VIADDMNMX.RELU + 1 IMAD per element, 3 PRMT per four.
__device__ __forceinline__ uint32_t norm_pack4(uint32_t x0, uint32_t x1, uint32_t x2, uint32_t x3, const NormCoef &c) {
    uint32_t z0, z1, z2, z3;
    // mul.lo via asm so the power-of-two multiply stays an IMAD (FMA pipe) instead of a shift on the ALU pipe
    asm("mul.lo.u32 %0, %1, %2;" : "=r"(z0) : "r"((uint32_t)__viaddmin_s32_relu((int)x0, c.rounding, c.cap)), "r"(c.mult));
    asm("mul.lo.u32 %0, %1, %2;" : "=r"(z1) : "r"((uint32_t)__viaddmin_s32_relu((int)x1, c.rounding, c.cap)), "r"(c.mult));
    asm("mul.lo.u32 %0, %1, %2;" : "=r"(z2) : "r"((uint32_t)__viaddmin_s32_relu((int)x2, c.rounding, c.cap)), "r"(c.mult));
    asm("mul.lo.u32 %0, %1, %2;" : "=r"(z3) : "r"((uint32_t)__viaddmin_s32_relu((int)x3, c.rounding, c.cap)), "r"(c.mult));
    uint32_t lo = __byte_perm(z0, z1, 0x0073), hi = __byte_perm(z2, z3, 0x0073);
    return __byte_perm(lo, hi, 0x5410);
}

// ---------------------------------------------------------------------------------------------------
// the kernel
//
// Roles (one CTA per SM, persistent over image tiles):
//   * kPipes x 2 consumer warpgroups.  Warpgroup 2p + h takes rows 64h .. 64h+63 of every tile of pipe p (tiles i of this CTA with
//     i % kPipes == p) and runs the whole layer chain on them in registers.
//   * one producer warp: barrier setup, the weight copy, and (int8 input) the TMA image loads of every pipe in tile order.
//   * kFloatIn: eight quantiser warps in place of the TMA loads (see below).
// Barriers: full[stage] (tile landed: TMA bytes, or the eight quantiser warps), empty[stage] (the eight consumer warps of the pipe
// have finished reading the stage).  Every consumer and the producer visit the stages of their pipe in order, so every parity
// wait starts after the barrier's previous phase has completed: one full and one empty barrier per stage suffice.
// ---------------------------------------------------------------------------------------------------
// 256-wide models: 128 accumulator + 32 fragment registers per consumer thread do not fit the 168 registers a 288-thread CTA
// gets, so the producer becomes a whole warpgroup that hands registers to the consumers (setmaxnreg: 2 x 128 x 224 + 128 x 56
// <= 64 k)
template <int kN, int kPipes, bool kFloatIn>
constexpr int chain_threads() { return (kN == 256 ? 384 : kPipes * 256 + 32) + (kFloatIn ? 32 * kFloatQuantWarps : 0); }

template <int kN, int kPipes, bool kFloatIn>
__global__ void __launch_bounds__(chain_threads<kN, kPipes, kFloatIn>(), 1)
fc_chain_kernel(const __grid_constant__ CUtensorMap tmap_in, const __grid_constant__ ChainParams P) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t bar_full[kMaxStages], bar_empty[kMaxStages];
    __shared__ __align__(8) uint64_t bar_w;   // weight image landed (bulk async copies)
    __shared__ __align__(8) uint64_t bar_fload[kFloatQuantWarps][2];   // kFloatIn: a quantiser warp's ring slot has landed

    const uint32_t tid = threadIdx.x, lane = tid & 31;
    const uint32_t warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
    // Programmatic dependent launch: the next kernel in the stream may take over each SM as soon as this CTA leaves it (it cannot
    // co-reside: every launch asks for more than half of the SM's shared memory), so its launch latency and prologue -- and, when
    // the caller declares consecutive launches independent, its first tiles -- overlap the ragged end of this one.  Only when the
    // grid fills the GPU: a smaller grid leaves SMs free, where later launches could pile up next to earlier ones.
    if (P.early_trigger) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const uint32_t n_st = P.n_stages;
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // SWIZZLE_128B tiles need 1024-byte alignment
    uint8_t *smem = smem_raw + (smem_base - smem_u32(smem_raw));

    const uint32_t tile0 = blockIdx.x, tile_step = gridDim.x;
    const uint32_t my_tiles = tile0 < P.n_tiles ? (P.n_tiles - tile0 + tile_step - 1) / tile_step : 0;
    const uint32_t w_base = smem_base + P.off_w;
    const uint32_t prod_warp = kPipes * 8;
    // tile i of this CTA: pipe i % kPipes, j-th tile of that pipe, stage (pipe, j % n_st), ring round j / n_st
    auto stage_of = [&](uint32_t i) { return (i % kPipes) * n_st + (i / kPipes) % n_st; };
    auto round_of = [&](uint32_t i) { return (i / kPipes) / n_st; };

    if (warp == prod_warp) {
        if (lane < kPipes * n_st) {
            mbar_init(&bar_full[lane], kFloatIn ? kFloatQuantWarps : 1);
            mbar_init(&bar_empty[lane], kEmptyArrivals);
        }
        if (lane == 31) mbar_init(&bar_w, 1);
        if (kFloatIn && lane >= 8 && lane < 8 + 2 * kFloatQuantWarps) mbar_init(&bar_fload[(lane - 8) >> 1][lane & 1], 1);
        fence_mbar_init();
        __syncwarp();
    }
    __syncthreads();

    if (warp == prod_warp || (kN == 256 && warp > prod_warp)) {
        // ======================= producer (256-wide: its whole warpgroup gives registers away, three warps of it idle) ============
        if (kN == 256) asm volatile("setmaxnreg.dec.sync.aligned.u32 56;" ::: "memory");
        if (warp == prod_warp && lane == 0) {
            // weight image -> smem (same bytes for every CTA; L2-resident after the first wave).  The weights were written at model
            // build, long before any kernel that may still be running ahead of this one, so they are fetched before the grid
            // dependency is resolved.
            mbar_arrive_expect_tx(&bar_w, P.w_bytes);
            for (uint32_t off = 0; off < P.w_bytes; off += 32768)
                bulk_load_1d(smem + P.off_w + off, P.w_image + off, min(32768u, P.w_bytes - off), &bar_w);
            if (!kFloatIn) {
                // everything else this kernel reads or writes may belong to the kernel launched before it
                if (P.wait_prior_grid) asm volatile("griddepcontrol.wait;" ::: "memory");
                const uint64_t l2_policy = policy_evict_first();   // images are read exactly once
                for (uint32_t i = 0; i < my_tiles; i++) {
                    const uint32_t s = stage_of(i), u = round_of(i);
                    if (u > 0) mbar_wait_relaxed(&bar_empty[s], (u - 1) & 1, P.err, 5);
                    mbar_arrive_expect_tx(&bar_full[s], P.stage_bytes);
                    const int32_t row = (int32_t)((tile0 + i * tile_step) * kTileM);
                    for (uint32_t a = 0; a < P.in_atoms; a++)
                        tma_load_2d_hint(smem + s * P.stage_bytes + a * 16384, &tmap_in, (int32_t)(a * 128), row, &bar_full[s], l2_policy);
                }
            }
        }
    } else if (warp < prod_warp) {
        // ======================= consumer warpgroup cw = 2 pipe + half =======================
        if (kN == 256) asm volatile("setmaxnreg.inc.sync.aligned.u32 224;" ::: "memory");
        const uint32_t cw = warp >> 2, pipe = cw >> 1, half = cw & 1, wq = warp & 3;
        const uint32_t quad = lane & 3;
        const uint32_t row_in_tile = half * 64 + wq * 16 + (lane >> 2);   // this thread's first row; the second is 8 below
        const int n_layers = P.n_layers;
        const uint32_t ncls = P.n_classes;
        mbar_wait(&bar_w, 0, P.err, 6);   // weight tiles are in shared memory
        // B descriptor of the 64 columns from c0 of the K-step tile at smem address t (no-swizzle K-major: 8-row groups 256 B apart).
        // Every wgmma is issued at the kernel's full width kN, with no condition around it (a conditional wgmma cannot stay in
        // the asynchronous pipeline): columns past a layer's n_pad and K-steps past its k_steps read the zero tile at w_zero
        // instead (a piece that straddles n_pad reads up to 48 rows past its tile, which the zero tile behind the image also
        // covers); the epilogue ignores those columns.
        const uint32_t w_zero = w_base + P.zero_off;
        auto b_desc = [](uint32_t t, int c0) { return make_smem_desc(t + (uint32_t)c0 / 8 * 256, 128, 256, GMMA_LAYOUT_NONE); };
        uint32_t acc[kN / 2];
        uint32_t afr[kN / 8];          // next layer's A fragments: 4 registers per K-step of 32
#pragma unroll 1
        for (uint32_t i = pipe; i < my_tiles; i += kPipes) {
            const uint32_t s = stage_of(i);
            mbar_wait(&bar_full[s], round_of(i) & 1, P.err, 2);
            // ---- layer 1 (A: the SW128 image stage, this warpgroup's 64 rows start 8 KB in for the lower half)
            {
                const uint64_t a0 = make_smem_desc(smem_base + s * P.stage_bytes + half * 8192, 16, 1024, GMMA_LAYOUT_SW128);
                const uint32_t n_pad = P.n_pad[0], k_steps = P.k_steps[0];
                wgmma_fence();
#pragma unroll 1
                for (uint32_t pl = 0; pl < P.planes[0]; pl++)
#pragma unroll 1
                    for (uint32_t k = 0; k < k_steps; k++) {
                        // K advance inside a SW128 atom: +32 B (>>4 = 2); next atom: +16384 B (>>4 = 1024).  B: +n_pad x 32 B per K-step
                        const uint64_t ad = a0 + (uint64_t)((k >> 2) * 1024 + (k & 3) * 2);
                        const uint32_t bt = w_base + P.b_off[0] + (pl * k_steps + k) * n_pad * 32;
#pragma unroll
                        for (int c0 = 0; c0 < kN; c0 += 64)
                            wgmma_ss_n64(acc + c0 / 2, ad, b_desc((uint32_t)c0 < n_pad ? bt : w_zero, c0), (pl | k) != 0);
                    }
                wgmma_commit();
                wgmma_wait<0>();
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&bar_empty[s]);   // this warp's reads of the stage are complete
            for (int l = 0;; l++) {
                const uint32_t n_pad = P.n_pad[l];
                if (l + 1 < n_layers) {
                    // ---- ReLUNorm of layer l into the A fragments of layer l + 1
                    int m0 = 0, m1 = 0;
#pragma unroll
                    for (int j = 0; j < kN / 8; j += 2)
                        if ((uint32_t)j * 8 < n_pad) {
                            m0 = __vimax3_s32(m0, (int)acc[4 * j], (int)acc[4 * j + 1]);
                            m1 = __vimax3_s32(m1, (int)acc[4 * j + 2], (int)acc[4 * j + 3]);
                            m0 = __vimax3_s32(m0, (int)acc[4 * j + 4], (int)acc[4 * j + 5]);
                            m1 = __vimax3_s32(m1, (int)acc[4 * j + 6], (int)acc[4 * j + 7]);
                        }
                    m0 = max(m0, __shfl_xor_sync(0xffffffffu, m0, 1));
                    m1 = max(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
                    m0 = max(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
                    m1 = max(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
                    const NormCoef k0 = norm_coef(m0), k1 = norm_coef(m1);
                    // 16-column block b -> register 2b (upper row) / 2b + 1 (lower row) of the fragments, i.e. for K-step s = b / 2:
                    // a[4s] (upper row, block 2s), a[4s + 1] (lower, 2s), a[4s + 2] (upper, 2s + 1), a[4s + 3] (lower, 2s + 1)
#pragma unroll
                    for (int b = 0; b < kN / 16; b++) {
                        const int f = 4 * (b >> 1) + 2 * (b & 1);
                        if ((uint32_t)b * 16 < n_pad) {
                            afr[f] = norm_pack4(acc[8 * b], acc[8 * b + 1], acc[8 * b + 4], acc[8 * b + 5], k0);
                            afr[f + 1] = norm_pack4(acc[8 * b + 2], acc[8 * b + 3], acc[8 * b + 6], acc[8 * b + 7], k1);
                        } else {
                            afr[f] = 0;
                            afr[f + 1] = 0;
                        }
                    }
                    // ---- layer l + 1 (A: registers)
                    const uint32_t n_next = P.n_pad[l + 1], k_steps = P.k_steps[l + 1], b_l = w_base + P.b_off[l + 1];
                    wgmma_fence();
#pragma unroll 1
                    for (uint32_t pl = 0; pl < P.planes[l + 1]; pl++)
#pragma unroll
                        for (int k = 0; k < kN / 32; k++) {   // unrolled: the fragment index stays a compile-time constant
                            const uint32_t bt = (uint32_t)k < k_steps ? b_l + (pl * k_steps + k) * n_next * 32 : w_zero;
#pragma unroll
                            for (int c0 = 0; c0 < kN; c0 += 64)
                                wgmma_rs_n64(acc + c0 / 2, afr + 4 * k, b_desc((uint32_t)c0 < n_next ? bt : w_zero, c0), (pl | k) != 0);
                        }
                    wgmma_commit();
                    wgmma_wait<0>();
                    continue;
                }
                // ---- logits + label (dll.c:115-116: the last ReLUNorm's argmax is what Inference() returns).  argmax = first
                // maximum (strict '>' from -INT32_MAX, pos 255, inference.c:32-37): in column order per thread, then over the quad
                const uint32_t tile = tile0 + i * tile_step;
#pragma unroll
                for (int r = 0; r < 2; r++) {
                    const size_t img = (size_t)tile * kTileM + row_in_tile + 8 * r;
                    int best = -INT32_MAX;
                    uint32_t pos = 255;
#pragma unroll
                    for (int j = 0; j < kN / 8; j++)
#pragma unroll
                        for (int e = 0; e < 2; e++) {
                            const uint32_t col = 8 * j + 2 * quad + e;
                            const int x = (int)acc[4 * j + 2 * r + e];
                            if (col < ncls && x > best) { best = x; pos = col; }
                        }
#pragma unroll
                    for (int sh = 1; sh <= 2; sh <<= 1) {
                        const int ob = __shfl_xor_sync(0xffffffffu, best, sh);
                        const uint32_t op = __shfl_xor_sync(0xffffffffu, pos, sh);
                        if (ob > best || (ob == best && op < pos)) { best = ob; pos = op; }
                    }
                    if (img < P.n) {
                        auto store_row = [&](int32_t *d) {
#pragma unroll
                            for (int j = 0; j < kN / 8; j++) {
                                const uint32_t col = 8 * j + 2 * quad;
                                if ((ncls & 1) == 0) {   // rows are 8-byte aligned: 64-bit stores
                                    if (col < ncls) *reinterpret_cast<int2 *>(d + col) = make_int2((int)acc[4 * j + 2 * r], (int)acc[4 * j + 2 * r + 1]);
                                } else {
                                    if (col < ncls) d[col] = (int)acc[4 * j + 2 * r];
                                    if (col + 1 < ncls) d[col + 1] = (int)acc[4 * j + 2 * r + 1];
                                }
                            }
                        };
                        store_row(P.logits + img * ncls);
#pragma unroll 1
                        for (uint32_t d = 0; d < P.n_log_dst; d++) store_row(P.log_dst[d] + (P.row0 + img) * ncls);   // peers, over NVLink
                        if (quad == 0) {
                            if (P.labels) P.labels[img] = pos;
#pragma unroll 1
                            for (uint32_t d = 0; d < P.n_lab_dst; d++) {
                                if (P.lab_u8) reinterpret_cast<uint8_t *>(P.lab_dst[d])[P.row0 + img] = (uint8_t)pos;
                                else P.lab_dst[d][P.row0 + img] = pos;
                            }
                        }
                    }
                }
                break;
            }
        }
    } else if (kFloatIn) {
        // ======================= quantiser warps (float input): warp qw converts rows 16 qw .. 16 qw + 15 of every tile =======================
        // The input scaling of the reference's caller (test_inference.py:140-141: scale = 127 / max(max|x|, 1e-5), q = round-half-even
        // (x * scale) clipped to int8, all float32) is fused into the load stage.  The float rows of a warp's share are contiguous in
        // HBM: they are fetched four rows (4 kB) at a time by one bulk async copy into the warp's own two-slot ring.  A pass converts
        // four rows at once, eight lanes per row: a lane holds 32 of its row's floats (eight float4, visited in an order rotated by
        // the row so that the four rows never meet in a bank), so the row maximum needs three shuffles and every lane has 32
        // independent elements to scale, round and pack.  The int8 words go straight into the image stage the layer-1 MMA reads, in
        // its SWIZZLE_128B layout -- the place of the TMA load.
        if (P.wait_prior_grid) asm volatile("griddepcontrol.wait;" ::: "memory");
        const uint32_t qw = warp - prod_warp - 1;
        const uint32_t elems = P.in_elems, n_f4 = elems >> 2, row_words = P.in_atoms * 32;   // float4 per float row, 4-byte words per int8 row
        const float *src = P.fimages;
        uint8_t *ring = smem + P.off_fring + qw * (2 * kFloatGroupRows * 1024);
        uint64_t *fbar = &bar_fload[qw][0];
        constexpr uint32_t kGroupsPerTile = kFloatRowsPerWarp / kFloatGroupRows;
        const uint32_t n_groups = my_tiles * kGroupsPerTile;   // groups of rows of this warp, in order
        auto group_rows = [&](uint32_t gi, size_t &row) {   // first global row and number of valid rows of group gi
            const uint32_t i = gi / kGroupsPerTile, k = gi % kGroupsPerTile;
            row = (size_t)(tile0 + i * tile_step) * kTileM + qw * kFloatRowsPerWarp + k * kFloatGroupRows;
            return row < P.n ? (uint32_t)min((size_t)kFloatGroupRows, P.n - row) : 0u;
        };
        auto issue_group = [&](uint32_t gi) {
            size_t row;
            const uint32_t valid = group_rows(gi, row);
            if (lane == 0 && valid) {
                mbar_arrive_expect_tx(&fbar[gi & 1], valid * elems * 4);
                bulk_load_1d(ring + (gi & 1) * (kFloatGroupRows * 1024), src + row * elems, valid * elems * 4, &fbar[gi & 1]);
            }
        };
        const uint32_t u = lane >> 3, sub = lane & 7;   // row of the pass, position inside the row's eight-lane team
        uint32_t fphase = 0;   // one phase bit per ring slot
        if (n_groups > 0) issue_group(0);
        if (n_groups > 1) issue_group(1);
        for (uint32_t gi = 0; gi < n_groups; gi++) {
            const uint32_t i = gi / kGroupsPerTile, k = gi % kGroupsPerTile, s = stage_of(i), rnd = round_of(i);
            if (k == 0 && rnd > 0) mbar_wait(&bar_empty[s], (rnd - 1) & 1, P.err, 8);   // the tile that used this stage is through layer 1
            uint8_t *stage = smem + s * P.stage_bytes;
            size_t row;
            const uint32_t valid = group_rows(gi, row);
            const uint32_t slot = gi & 1;
            if (valid) {
                mbar_wait(&fbar[slot], (fphase >> slot) & 1, P.err, 9);
                fphase ^= 1u << slot;
            }
            const float4 *fr = reinterpret_cast<const float4 *>(ring + slot * (kFloatGroupRows * 1024)) + u * n_f4;
            const uint32_t r = qw * kFloatRowsPerWarp + k * kFloatGroupRows + u;   // this lane's row inside the tile
            float4 v[8];
            float m = 0.f;
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const uint32_t c = sub + 8 * ((j + u) & 7);
                v[j] = (u < valid && c < n_f4) ? fr[c] : make_float4(0.f, 0.f, 0.f, 0.f);
                m = fmaxf(m, fmaxf(fmaxf(fabsf(v[j].x), fabsf(v[j].y)), fmaxf(fabsf(v[j].z), fabsf(v[j].w))));
            }
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 4));
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
            m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
            // test_inference.py:140-141 / BitNetMCU.py:435-436, every step one correctly rounded float32 operation
            const float scale = __fdiv_rn(127.0f, fmaxf(m, 1e-5f));
            auto q = [&](float x) { int d; asm("cvt.rni.sat.s8.f32 %0, %1;" : "=r"(d) : "f"(__fmul_rn(x, scale))); return (uint32_t)d; };   // round half to even, clip to int8
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const uint32_t c = sub + 8 * ((j + u) & 7);   // word c of the int8 row (bytes 4c .. 4c+3)
                const uint32_t w = __byte_perm(__byte_perm(q(v[j].x), q(v[j].y), 0x0040), __byte_perm(q(v[j].z), q(v[j].w), 0x0040), 0x5410);
                // SWIZZLE_128B: 16-byte chunk jc of row r sits at chunk position jc ^ (r & 7) of the row's 128 bytes in its atom
                if (c < row_words)
                    *reinterpret_cast<uint32_t *>(stage + (c >> 5) * 16384 + r * 128 + ((((c & 31) >> 2) ^ (r & 7)) << 4) + (c & 3) * 4) = w;
            }
            __syncwarp();   // every lane has read its floats of this slot
            if (gi + 2 < n_groups) issue_group(gi + 2);
            if (k == kGroupsPerTile - 1) {
                fence_proxy_async_smem();   // the layer-1 MMAs (async proxy) read what these generic-proxy stores wrote
                __syncwarp();
                if (lane == 0) mbar_arrive(&bar_full[s]);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

static uint32_t round_up(uint32_t v, uint32_t m) { return (v + m - 1) / m * m; }

template <int kN, int kPipes, bool kFloatIn>
static cudaError_t launch_chain(const cudaLaunchConfig_t &cfg, const CUtensorMap &tmap, const ChainParams &p) {
    return cudaLaunchKernelEx(&cfg, fc_chain_kernel<kN, kPipes, kFloatIn>, tmap, p);
}
template <int kN, int kPipes, bool kFloatIn>
static bool opt_in_smem(int bytes) {
    return cudaFuncSetAttribute(fc_chain_kernel<kN, kPipes, kFloatIn>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) == cudaSuccess;
}

static cudaError_t dispatch(const FcChainPlan *plan, bool float_in, const cudaLaunchConfig_t &cfg, const CUtensorMap &tmap, const ChainParams &p) {
    if (float_in) return launch_chain<64, 1, true>(cfg, tmap, p);   // plans of wider models have no float-input form
    if (plan->max_n == 64) return plan->pipes == 2 ? launch_chain<64, 2, false>(cfg, tmap, p) : launch_chain<64, 1, false>(cfg, tmap, p);
    if (plan->max_n == 128) return launch_chain<128, 1, false>(cfg, tmap, p);
    if (plan->max_n == 192) return launch_chain<192, 1, false>(cfg, tmap, p);
    return launch_chain<256, 1, false>(cfg, tmap, p);
}

FcChainPlan *fc_chain_plan_create(const FcLayerDev *layers, int n_layers, uint32_t in_bytes, int device, int sm_count,
                                  char *err, size_t err_len) {
    auto fail = [&](const char *msg) -> FcChainPlan * { if (err) snprintf(err, err_len, "%s", msg); return nullptr; };
    if (n_layers < 1 || n_layers > kMaxFcLayers) return fail("fused path: 1..8 FC layers");
    if (in_bytes % 16 || in_bytes == 0 || in_bytes > 1024) return fail("fused path: input row must be a multiple of 16 bytes, <= 1024");
    if (!get_encode_fn()) return fail("cuTensorMapEncodeTiled not available");
    auto *plan = new FcChainPlan();
    ChainParams &p = plan->p;
    p.n_layers = n_layers;
    p.in_atoms = (in_bytes + 127) / 128;   // weights past the real input width multiply zero activations: dropped
    p.stage_bytes = p.in_atoms * 16384;
    uint32_t w_off = 0, max_n = 0;
    for (int l = 0; l < n_layers; l++) {
        const FcLayerDev &L = layers[l];
        if (L.n_pad > 256) { delete plan; return fail("fused path: layer wider than 256 outputs"); }
        p.n_pad[l] = L.n_pad;
        // K of layer l > 0: the activations past the previous layer's (padded) width are zero -- e.g. Ternary pads n_in to a
        // multiple of 10 with zero trits (64 -> 70, exportquant.py:132-137) -- so those K-steps are dropped, exactly
        p.k_steps[l] = l == 0 ? p.in_atoms * 4 : round_up(std::min(L.k_pad, layers[l - 1].n_pad), 32) / 32;
        p.planes[l] = L.dense_b ? 2 : 1;
        p.b_off[l] = w_off;
        w_off += p.planes[l] * p.k_steps[l] * L.n_pad * 32;
        max_n = std::max(max_n, L.n_pad);
    }
    // the kernel's accumulator width: the widest layer rounded up to the 64-column wgmma pieces.  Accumulator registers per thread
    // = max_n / 2.  Two pipes (four consumer warpgroups, 544 threads: up to five warps share an SM sub-partition, <= 96 registers
    // each) only for models up to 64 wide; wider ones run one pipe (288 threads, <= 168 registers)
    plan->max_n = round_up(max_n, 64);
    p.zero_off = w_off;                    // [max_n x 32 B] of zeros behind the layers (cudaMemset below)
    p.w_bytes = w_off + plan->max_n * 32;
    p.n_classes = layers[n_layers - 1].n_out;
    const uint32_t smem_limit = 227 * 1024 - 1024 /*alignment slack*/ - 1024 /*static: barriers*/;
    const uint32_t w_fixed = round_up(p.w_bytes, 128);
    if (w_fixed + 2 * p.stage_bytes > smem_limit) { delete plan; return fail("fused path: weights do not fit in shared memory"); }
    const uint32_t total_stages = std::min<uint32_t>(kMaxStages, (smem_limit - w_fixed) / p.stage_bytes);
    plan->pipes = (plan->max_n == 64 && total_stages >= 4) ? 2 : 1;
    p.n_stages = std::min<uint32_t>(total_stages / plan->pipes, 6);
    p.off_w = plan->pipes * p.n_stages * p.stage_bytes;
    // One CTA per SM is part of the launch-overlap contract (launch k+2 must never run next to launch k on an SM): shared memory
    // enforces it once a CTA asks for more than half of the SM's 227 kB.
    plan->smem_bytes = std::max<size_t>((size_t)p.off_w + w_fixed + 1024, 116 * 1024);
    // float-input path: the eight quantiser warps make 17 warps, so at most 96 registers per thread -- models up to 64 wide
    if (in_bytes <= 256 && p.n_classes <= 16 && plan->max_n == 64) {
        const uint32_t fring = kFloatQuantWarps * 2 * kFloatGroupRows * 1024;
        const uint32_t fixed_f = w_fixed + fring;
        if (fixed_f + 2 * p.stage_bytes <= smem_limit) {
            plan->f_n_stages = std::min<uint32_t>(4, (smem_limit - fixed_f) / p.stage_bytes);
            plan->f_off_w = plan->f_n_stages * p.stage_bytes;
            plan->f_off_fring = plan->f_off_w + w_fixed;
            plan->f_smem_bytes = std::max<size_t>((size_t)plan->f_off_fring + fring + 1024, 116 * 1024);
        }
    }
    if (getenv("BNM_VERBOSE"))   // diagnostics: the shapes this plan launches
        fprintf(stderr, "bitnetmcu_b200: fused FC plan: %u accumulator columns, %u pipes x %u stages, %u weight bytes, %zu B smem\n",
                plan->max_n, plan->pipes, p.n_stages, p.w_bytes, plan->smem_bytes);
    plan->in_bytes = in_bytes;
    plan->sm_count = sm_count;
    plan->device = device;

    // weight image
    if (cudaMalloc(&plan->d_w_image, p.w_bytes) != cudaSuccess || cudaHostAlloc(&plan->h_err, sizeof(int), cudaHostAllocMapped) != cudaSuccess ||
        cudaHostGetDevicePointer(&plan->d_err, plan->h_err, 0) != cudaSuccess) {
        fc_chain_plan_destroy(plan);
        return fail("cudaMalloc failed (weight image)");
    }
    cudaMemset(plan->d_w_image, 0, p.w_bytes);
    *plan->h_err = 0;
    for (int l = 0; l < n_layers; l++) {
        const FcLayerDev &L = layers[l];
        for (uint32_t pl = 0; pl < p.planes[l]; pl++) {
            size_t total = (size_t)L.n_pad * p.k_steps[l] * 32;
            k_build_b_image<<<(unsigned)((total + 255) / 256), 256>>>(pl ? L.dense_b : L.dense_a, L.k_pad, L.n_pad, p.k_steps[l], l > 0,
                                                                      plan->d_w_image + p.b_off[l] + (size_t)pl * p.k_steps[l] * L.n_pad * 32);
        }
    }
    if (cudaDeviceSynchronize() != cudaSuccess) { fc_chain_plan_destroy(plan); return fail("weight image kernel failed"); }
    p.w_image = plan->d_w_image;
    p.err = plan->d_err;
    const int smem_any = (int)std::max(plan->smem_bytes, plan->f_smem_bytes);
    if (!opt_in_smem<64, 1, false>(smem_any) || !opt_in_smem<64, 2, false>(smem_any) || !opt_in_smem<128, 1, false>(smem_any) ||
        !opt_in_smem<192, 1, false>(smem_any) || !opt_in_smem<256, 1, false>(smem_any) || !opt_in_smem<64, 1, true>(smem_any)) {
        fc_chain_plan_destroy(plan);
        return fail("cannot opt in to the required dynamic shared memory");
    }
    return plan;
}

void fc_chain_plan_set_overlap(FcChainPlan *p, int mode) {
    if (!p) return;
    p->overlap = mode;
    p->prev_valid = false;
}

void fc_chain_plan_destroy(FcChainPlan *p) {
    if (!p) return;
    if (p->d_w_image) cudaFree(p->d_w_image);
    if (p->h_err) {
        if (*p->h_err) fprintf(stderr, "bitnetmcu_b200: fused FC kernel: bounded wait %d timed out (device trap)\n", *p->h_err);
        cudaFreeHost(p->h_err);
    }
    delete p;
}

static const CUtensorMap *plan_tensor_map(FcChainPlan *plan, const int8_t *in, size_t n) {
    for (auto &t : plan->tmaps)
        if (t.ptr == in && t.n == n) return &t.map;
    FcChainPlan::TmapSlot &t = plan->tmaps[plan->tmap_next++ % 4];
    memset(&t.map, 0, sizeof(t.map));
    cuuint64_t gdim[2] = {(cuuint64_t)plan->in_bytes, (cuuint64_t)n};
    cuuint64_t gstride[1] = {(cuuint64_t)plan->in_bytes};
    cuuint32_t box[2] = {128, (cuuint32_t)kTileM};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = get_encode_fn()(&t.map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<int8_t *>(in), gdim, gstride, box, estr,
                                 CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                 CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { t.ptr = nullptr; t.n = 0; return nullptr; }
    t.ptr = in;
    t.n = n;
    return &t.map;
}

int fc_chain_launch(FcChainPlan *plan, const int8_t *in, size_t n, int32_t *logits, uint32_t *labels, const GatherDst *gather,
                    cudaStream_t st) {
    if (n == 0) return 0;
    if (n > 0x7fffff00ull) return -2;
    ChainParams p = plan->p;
    p.logits = logits;
    p.labels = labels;
    p.n = n;
    p.n_lab_dst = p.n_log_dst = 0;
    p.row0 = 0;
    p.lab_u8 = 0;
    if (gather) {
        if (gather->n_labels_dst > (uint32_t)kMaxGatherDst || gather->n_logits_dst > (uint32_t)kMaxGatherDst) return -5;
        p.n_lab_dst = gather->n_labels_dst;
        p.n_log_dst = gather->n_logits_dst;
        p.row0 = gather->row_offset;
        p.lab_u8 = gather->labels_u8 && p.n_classes <= 255;
        if (gather->labels_u8 && !p.lab_u8) return -5;
        for (uint32_t d = 0; d < p.n_lab_dst; d++) p.lab_dst[d] = gather->labels_dst[d];
        for (uint32_t d = 0; d < p.n_log_dst; d++) p.log_dst[d] = gather->logits_dst[d];
    }
    p.n_tiles = (uint32_t)((n + kTileM - 1) / kTileM);
    const CUtensorMap *tmap_p = plan_tensor_map(plan, in, n);
    if (!tmap_p) return -3;
    const unsigned grid = (unsigned)std::min<uint32_t>(p.n_tiles, (uint32_t)plan->sm_count);
    // Mode 2 drops the grid-dependency wait, i.e. EVERY ordering against the work enqueued before this launch on the stream
    // (the previous bnm launch and any producer kernel of `images` alike).  The library keeps the wait whenever it can see the
    // promise being broken: first launch on this plan / another stream / a buffer of the previous launch reused.
    bool independent = plan->overlap == 2 && plan->prev_valid && plan->prev_stream == st && in != plan->prev_in &&
                       logits != plan->prev_logits && (labels == nullptr || labels != plan->prev_labels);
    p.wait_prior_grid = !independent;
    p.early_trigger = plan->overlap != 0 && grid == (unsigned)plan->sm_count;
    plan->prev_in = in; plan->prev_logits = logits; plan->prev_labels = labels; plan->prev_stream = st; plan->prev_valid = true;
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(plan->max_n == 256 ? 384 : plan->pipes * 256 + 32);   // chain_threads()
    cfg.dynamicSmemBytes = plan->smem_bytes;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = plan->overlap ? 1 : 0;
    if (dispatch(plan, false, cfg, *tmap_p, p) != cudaSuccess) return -4;
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

bool fc_chain_float_input_supported(const FcChainPlan *plan) {
    return plan && plan->f_smem_bytes != 0 && plan->in_bytes % 16 == 0;
}

// float32 images [n][in_bytes elements] -> logits / labels, the input scaling fused into the load stage (kFloatIn)
int fc_chain_launch_f32(FcChainPlan *plan, const float *in, size_t n, int32_t *logits, uint32_t *labels, cudaStream_t st) {
    if (n == 0) return 0;
    if (n > 0x7fffff00ull) return -2;
    if (!fc_chain_float_input_supported(plan)) return -6;
    ChainParams p = plan->p;
    p.logits = logits;
    p.labels = labels;
    p.n = n;
    p.n_lab_dst = p.n_log_dst = 0;
    p.row0 = 0;
    p.lab_u8 = 0;
    p.fimages = in;
    p.in_elems = plan->in_bytes;
    p.n_stages = plan->f_n_stages;
    p.off_w = plan->f_off_w;
    p.off_fring = plan->f_off_fring;
    p.n_tiles = (uint32_t)((n + kTileM - 1) / kTileM);
    p.wait_prior_grid = 1;
    p.early_trigger = 0;
    CUtensorMap tmap;   // not used by the float-input kernel (no TMA image loads)
    memset(&tmap, 0, sizeof(tmap));
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)std::min<uint32_t>(p.n_tiles, (uint32_t)plan->sm_count));
    cfg.blockDim = dim3(256 + 32 + 32 * kFloatQuantWarps);   // two consumer warpgroups + producer warp + the quantiser warps
    cfg.dynamicSmemBytes = plan->f_smem_bytes;
    cfg.stream = st;
    plan->prev_valid = false;
    if (dispatch(plan, true, cfg, tmap, p) != cudaSuccess) return -4;
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

}  // namespace bnm
