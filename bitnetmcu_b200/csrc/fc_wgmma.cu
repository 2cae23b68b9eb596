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
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "kernels.h"
#include "sm90_ptx.cuh"

namespace bnm {

constexpr int kMaxStages = 8;              // ring stages over all pipes of a CTA
constexpr uint32_t kEmptyArrivals = 8;     // a stage is free once the 8 warps of its two consumer warpgroups are past layer 1
constexpr uint32_t kFloatQuantWarps = 8;   // float-input path: quantiser warps per CTA (one pipe next to them)
constexpr uint32_t kFloatRowsPerWarp = 128 / kFloatQuantWarps;   // rows of every tile per quantiser warp
constexpr uint32_t kFloatGroupRows = 4;    // rows per bulk copy of a quantiser warp (4 kB for 256-element rows) = rows per pass

// What a launch form computes (the form table, host side below).  Rule: the hidden-layer rule -- the C engine's (inference.c),
// the reference's Python emulator's (emul_coef, float64 logits), or both on one tile (layer 1 once, its accumulators through
// both rules, then the C chain and the emulator's chain).  Outputs: logits and labels (the C engine on int8 rows also stores
// them to the result exchange's destinations); both engines' labels and their EngineTally counts; or the k best classes of
// every row and their scores, from k rounds of the epilogue's argmax.
enum FcRule { kRuleC, kRuleEmul, kRuleBoth };
enum FcOut { kOutLogits, kOutEngines, kOutTopK };

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
    // emulator launches (fc_emul_kernel): float64 logits [n][n_classes] (or null) = last layer's accumulators x logit_scale, the
    // emulator's 2^-level_shift of that layer's encoding (0.5 for 2bitsym / 4bitsym, else 1)
    double *emul_logits;
    double emul_logit_scale;
    // both-engine launches (fc_engines_kernel): `labels` are the C engine's, labels_py the emulator's; truth [n] and counts
    // (EngineTally's {images, correct_c, correct_py, mismatches}) may be null
    uint32_t *labels_py;
    const uint32_t *truth;
    unsigned long long *counts;
    // top-k launches (fc_topk_kernel): the k best classes of every row, uint32 [n][k], and their logits, int32 [n][k] (C engine)
    // or float64 [n][k] (emulator: accumulators x emul_logit_scale), or null; no logits, no labels, no result exchange
    uint32_t k;
    uint32_t *classes;
    int32_t *scores_i32;
    double *scores_f64;
};

struct ChainKernel;

// a launch form of a plan: its kernel row and its shared-memory layout, which every launch of the form copies into ChainParams
struct FormLayout {
    const ChainKernel *kernel = nullptr;   // null: the plan has no such form
    uint32_t n_stages = 0;                 // stages per pipe
    uint32_t off_w = 0, off_fring = 0;     // as in ChainParams; off_fring only for the float-input forms
    size_t smem_bytes = 0;                 // dynamic shared memory
};

// the device buffers one int8-form launch reads or writes, for the mode-2 check: images, logits and labels (null: none), and the
// gather destinations, which it writes from row row0 on
struct LaunchBuffers {
    const void *io[3] = {};
    const void *dst[2 * kMaxGatherDst] = {};
    uint32_t n_dst = 0;
    size_t row0 = 0;
};

// Does launch b touch a buffer of launch a?  Any non-null pointer of one equal to any of the other, whatever the roles, except
// that a destination both write counts only at the same row offset: the exchange's callers write their own rows of a shared
// destination, which the library cannot tell from overlapping ones (the caller's promise, like any aliasing at an offset).
static bool shares_buffer(const LaunchBuffers &a, const LaunchBuffers &b) {
    auto seen = [](const void *x, const void *const *set, uint32_t n) {
        for (uint32_t i = 0; i < n; i++)
            if (x && x == set[i]) return true;
        return false;
    };
    for (const void *x : b.io)
        if (seen(x, a.io, 3) || seen(x, a.dst, a.n_dst)) return true;
    for (uint32_t i = 0; i < b.n_dst; i++)
        if (seen(b.dst[i], a.io, 3) || (a.row0 == b.row0 && seen(b.dst[i], a.dst, a.n_dst))) return true;
    return false;
}

struct FcChainPlan {
    ChainParams p{};
    uint8_t *d_w_image = nullptr;
    int *d_err = nullptr;             // error word of the bounded device-side waits: mapped pinned host memory, readable after a trap
    int *h_err = nullptr;
    uint32_t in_bytes = 0;
    FormLayout forms[kFcForms];
    int sm_count = 0;
    int device = 0;
    int overlap = 0;                  // BNM_OPT_LAUNCH_OVERLAP: 0 and 1 dependent launch + wait, 2 independent launches
    struct TmapSlot { const void *ptr = nullptr; size_t n = 0; CUtensorMap map; };
    TmapSlot tmaps[4];                // tensor maps of the most recent (pointer, n) pairs: double/triple-buffered callers hit every time
    unsigned tmap_next = 0;
    // mode 2 bookkeeping: the buffers of the previous launch on this plan (the promise "consecutive launches are independent" is
    // checked as far as the library can see it: a launch that touches a buffer of the one before keeps the grid-dependency wait)
    LaunchBuffers prev;
    cudaStream_t prev_stream = nullptr;
    bool prev_valid = false;
    bool verbose = false;             // BNM_VERBOSE at plan creation: every int8-form launch names its wait decision
    // guards the tensor-map cache and the bookkeeping above together with the launch they describe: launches from several host
    // threads enqueue in the order the bookkeeping records
    std::mutex mu;
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
// The hidden-layer rule of the reference's Python emulator (BitNetMCU.py:452-457, restated in k_relunorm_emul) in registers:
//   out = round_half_even(relu(acc) * 2^e),  e = floor(log2(127 / m)),  m = row maximum;  m <= 0: the whole row is zero.
// The emulator divides acc by the level scale 2^ls before it takes the maximum and multiplies by 2^floor(log2(127 * 2^ls / m))
// after: the 2^ls cancels exactly, so e does not depend on the encoding.  With z = clz(m) (bit length 32 - z), m << z lies in
// [2^31, 2^32): e = z - 25, minus 1 when m << z exceeds 127 << 25.  m * 2^e <= 127, so the clip to 127 never triggers.
// Per element, with t = relu(v) * 2^max(e, 0) and s = max(-e, 0):  q = (t + 2^(s-1) - 1 + ((t >> s) & 1)) >> s  (round half to
// even; for s = 0 both addends are zero).  t < 2^31 and 2^(s-1) <= 2^24, so the unsigned sum does not wrap.
// ---------------------------------------------------------------------------------------------------
struct EmulCoef { uint32_t mult, s, bias, odd; };

__device__ __forceinline__ EmulCoef emul_coef(int row_max_relu) {
    const uint32_t m = (uint32_t)max(row_max_relu, 1);   // m = 0: every v <= 0, any e gives zeros -- take m = 1 (no shift by 32)
    const uint32_t z = __clz(m);
    const int e = (int)z - 25 - ((m << z) > (127u << 25) ? 1 : 0);
    EmulCoef c;
    c.mult = e > 0 ? 1u << e : 1u;
    c.s = e < 0 ? (uint32_t)-e : 0u;
    c.bias = c.s ? (1u << (c.s - 1)) - 1u : 0u;
    c.odd = c.s ? 1u : 0u;
    return c;
}
__device__ __forceinline__ uint32_t emul_q(uint32_t x, const EmulCoef &c) {
    uint32_t t;
    asm("mul.lo.u32 %0, %1, %2;" : "=r"(t) : "r"((uint32_t)max((int)x, 0)), "r"(c.mult));   // an IMAD, as in norm_pack4
    return (t + c.bias + ((t >> c.s) & c.odd)) >> c.s;
}
// four int32 accumulators -> four int8 (0..127) packed little-endian, emulator rule
__device__ __forceinline__ uint32_t norm_pack4(uint32_t x0, uint32_t x1, uint32_t x2, uint32_t x3, const EmulCoef &c) {
    return __byte_perm(__byte_perm(emul_q(x0, c), emul_q(x1, c), 0x0040), __byte_perm(emul_q(x2, c), emul_q(x3, c), 0x0040), 0x5410);
}

// ---------------------------------------------------------------------------------------------------
// phase trace (diagnostics build only: make -C bitnetmcu_b200/csrc EXTRA=-DBNM_FC_TRACE; tools/fc_phase_trace.py reads it).
// In the first kTraceCtas CTAs, lane 0 of warp 0 of every consumer warpgroup (writer cw) and the producer warp (writer
// kTraceWriters - 1) record (clock64, event) pairs; thread 0 records %globaltimer and clock64 at kernel entry and exit so that
// cycles convert to time.  The product build contains none of it.
// ---------------------------------------------------------------------------------------------------
#ifdef BNM_FC_TRACE
constexpr uint32_t kTraceCtas = 4, kTraceWriters = 5, kTraceEvents = 2048;
// event code: kind | slot << 8 | layer << 12
enum : uint32_t { TR_FULL_BEGIN = 1, TR_FULL_END, TR_WAIT_BEGIN, TR_WAIT_END, TR_EPI_END, TR_EMPTY_BEGIN, TR_EMPTY_END, TR_ISSUE };
struct FcTrace {
    unsigned long long hdr[kTraceCtas][4];   // globaltimer / clock64 at entry, globaltimer / clock64 at exit
    uint32_t count[kTraceCtas][kTraceWriters];
    ulonglong2 ev[kTraceCtas][kTraceWriters][kTraceEvents];   // (clock64, event code)
};
__device__ FcTrace g_fc_trace;
__device__ __forceinline__ unsigned long long globaltimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
#define BNM_TRACE_DECL(writer_, enabled_) const uint32_t tr_w = (writer_); const bool tr_on = (enabled_) && blockIdx.x < kTraceCtas; uint32_t tr_n = 0
#define BNM_TRACE(kind_, slot_, layer_) do { if (tr_on && tr_n < kTraceEvents) g_fc_trace.ev[blockIdx.x][tr_w][tr_n++] = make_ulonglong2((unsigned long long)clock64(), (kind_) | (uint32_t)(slot_) << 8 | (uint32_t)(layer_) << 12); } while (0)
#define BNM_TRACE_END() do { if (tr_on) g_fc_trace.count[blockIdx.x][tr_w] = tr_n; } while (0)
#define BNM_TRACE_STAMP(k_) do { if (threadIdx.x == 0 && blockIdx.x < kTraceCtas) { g_fc_trace.hdr[blockIdx.x][2 * (k_)] = globaltimer(); g_fc_trace.hdr[blockIdx.x][2 * (k_) + 1] = clock64(); } } while (0)
#else
#define BNM_TRACE_DECL(writer_, enabled_) do {} while (0)
#define BNM_TRACE(kind_, slot_, layer_) do {} while (0)
#define BNM_TRACE_END() do {} while (0)
#define BNM_TRACE_STAMP(k_) do {} while (0)
#endif

// ---------------------------------------------------------------------------------------------------
// the kernel
//
// Roles (one CTA per SM, persistent over image tiles):
//   * kPipes x 2 consumer warpgroups.  Warpgroup 2p + h takes rows 64h .. 64h+63 of every tile of pipe p (tiles i of this CTA with
//     i % kPipes == p) and runs the whole layer chain on them in registers.  With kSlots = 2 a warpgroup holds two consecutive tiles
//     of its pipe at once (slots A and B, each with its own accumulators and fragments) and alternates between them, so that the
//     MMAs of one slot are in flight while the warpgroup runs the ReLUNorm or the epilogue of the other.
//   * one producer warp: barrier setup, the weight copy, and (int8 input) the TMA image loads of every pipe in tile order.
//   * kFloatIn: eight quantiser warps in place of the TMA loads (see below).
// Barriers: full[stage] (tile landed: TMA bytes, or the eight quantiser warps), empty[stage] (the eight consumer warps of the pipe
// have finished reading the stage).  Every consumer and the producer visit the stages of their pipe in order, so every parity
// wait starts after the barrier's previous phase has completed: one full and one empty barrier per stage suffice.  Two slots keep
// that order: slot A waits for tile j, slot B for tile j + 1, and A's next tile j + 2 is waited for after both.
// ---------------------------------------------------------------------------------------------------
// The producer becomes a whole warpgroup that hands registers to the consumers (setmaxnreg) where the consumers need more than
// an even share of the register file.  setmaxnreg moves registers inside the CTA's launch allocation (threads x the per-thread
// count the launch bounds give), so the registers of all warps after it may not exceed that allocation:
//   * 256-wide models: 128 accumulator + 32 fragment registers per consumer thread do not fit the 168 registers a 288-thread CTA
//     gets; 384 threads x 168 = 2 x 128 x 224 + 128 x 56;
//   * two slots: 2 x (32 + 8) registers of accumulators and fragments per consumer thread do not fit the 96 a 544-thread CTA gets
//     (five warps on a sub-partition); 640 threads x 96 = 4 x 128 x 112 + 128 x 32.
template <int kN, int kSlots>
__host__ __device__ constexpr bool producer_warpgroup() { return kN == 256 || kSlots == 2; }
template <int kN, int kPipes, bool kFloatIn, int kSlots>
__host__ __device__ constexpr int chain_threads() {
    return kPipes * 256 + (producer_warpgroup<kN, kSlots>() ? 128 : 32) + (kFloatIn ? 32 * kFloatQuantWarps : 0);
}
// registers per thread of a one-CTA-per-SM launch of `threads`: the warps share four sub-partitions of 16 k registers each,
// allocated in steps of 8 per thread
__host__ __device__ constexpr int launch_regs(int threads) { return 16384 / (32 * ((threads / 32 + 3) / 4)) / 8 * 8; }

// The shape class of the fixed-shape kernel (kFixed): 256-byte input rows (two SW128 atoms, eight layer-1 K-steps), three
// 64-wide layers and a classes layer at most 16 wide, one weight plane each -- FC 4bitsym-64, Ternary-64 and the other 64-wide
// models.  Every layer's shape and its place in the weight image are compile-time constants of that kernel.
constexpr int kFixedLayers = 4;
constexpr uint32_t kFixedInAtoms = 2;
__host__ __device__ constexpr uint32_t fixed_n_pad(int l) { return l + 1 < kFixedLayers ? 64u : 16u; }
__host__ __device__ constexpr uint32_t fixed_k_steps(int l) { return l == 0 ? kFixedInAtoms * 4 : 2u; }
__host__ __device__ constexpr uint32_t fixed_b_off(int l) { return l == 0 ? 0u : fixed_b_off(l - 1) + fixed_k_steps(l - 1) * fixed_n_pad(l - 1) * 32; }
// a shared-memory descriptor advanced by `units` x 16 bytes: the 14-bit start field of an address inside the CTA's shared memory
// does not carry into the fields above it, so a 32-bit add of the low word is enough
__device__ __forceinline__ uint64_t desc_add(uint64_t d, uint32_t units) {
    return (d & 0xFFFFFFFF00000000ull) | (uint32_t)((uint32_t)d + units);
}

// Ring position of a pipe's next tile: its stage inside the pipe and the parity of its ring round.  Every role visits the tiles
// of a pipe in order and advances the position once per tile, so no role divides by the stage count.  Both live in one word:
// with two, the one-slot kernels need up to two more registers.
struct RingPos {
    uint32_t word = 0;   // stage | phase << 31
    __device__ __forceinline__ uint32_t stage() const { return word & 0x7fffffffu; }
    __device__ __forceinline__ uint32_t phase() const { return word >> 31; }
    __device__ __forceinline__ void advance(uint32_t n_st) {
        if ((++word & 0x7fffffffu) == n_st) word = (word & 0x80000000u) ^ 0x80000000u;
    }
};

// kSlots: tiles per consumer warpgroup in compute at once (1 or 2; 2 only for 64-wide int8 launches with two pipes).
// kLastN: wgmma width of the last layer -- 16 when the plan's last layer is at most 16 wide (every classifier head), else kN.
// kFixed: the two-slot kernel specialised for the shape class above: no plane loop, no zero-tile selects, layer 1 issued as
// one unrolled run of MMAs at compile-time descriptor offsets, ReLUNorm without predicates.
// kRule, kOut: the rule and the outputs of the launch form (the form table, host side below).
// The body of the kernels below; tmap_in and P are their __grid_constant__ parameters (TMA reads the tensor map by address).
template <int kN, int kPipes, bool kFloatIn, int kSlots, int kLastN, bool kFixed, FcRule kRule, FcOut kOut>
__device__ __forceinline__ void fc_chain_body(const CUtensorMap &tmap_in, const ChainParams &P) {
    static_assert(kSlots == 1 || (kSlots == 2 && kN == 64 && kPipes == 2 && !kFloatIn), "two slots: 64-wide int8 two-pipe launches");
    static_assert((kRule == kRuleC && kOut == kOutLogits) || (kPipes == 1 && kSlots == 1 && kLastN == kN && !kFixed),
                  "the emulator, both engines and top-k: one-pipe one-slot launches at full width");
    static_assert((kRule == kRuleBoth) == (kOut == kOutEngines), "both rules: the engines' outputs, which need both");
    static_assert(!kFloatIn || (kPipes == 1 && kN == 64),
                  "float input: one pipe, whose stages the quantiser warps fill; 17 warps leave 96 registers, enough for 64 wide");
    static_assert(kLastN == kN || (kLastN == 16 && kSlots == 2), "narrow last layer: two-slot launches");
    static_assert(!kFixed || (kSlots == 2 && kLastN == fixed_n_pad(kFixedLayers - 1)), "fixed shape: two-slot launches of its class");
    constexpr bool kProducerWG = producer_warpgroup<kN, kSlots>();
    constexpr uint32_t kProducerRegs = kN == 256 ? 56 : 32, kConsumerRegs = kN == 256 ? 224 : 112;
    static_assert(!kProducerWG || 128 * kProducerRegs + 256 * kPipes * kConsumerRegs <=
                  (uint32_t)(chain_threads<kN, kPipes, kFloatIn, kSlots>() * launch_regs(chain_threads<kN, kPipes, kFloatIn, kSlots>())),
                  "setmaxnreg: the warps' registers must fit the CTA's launch allocation, or an increase never returns");
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
    BNM_TRACE_STAMP(0);
    const uint32_t n_st = P.n_stages;
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // SWIZZLE_128B tiles need 1024-byte alignment
    uint8_t *smem = smem_raw + (smem_base - smem_u32(smem_raw));

    const uint32_t tile0 = blockIdx.x, tile_step = gridDim.x;
    const uint32_t my_tiles = tile0 < P.n_tiles ? (P.n_tiles - tile0 + tile_step - 1) / tile_step : 0;
    const uint32_t w_base = smem_base + P.off_w;
    const uint32_t prod_warp = kPipes * 8;
    // tile i of this CTA: pipe i % kPipes, j-th tile of that pipe, stage (pipe, j % n_st), ring round j / n_st.
    // Two slots: a warpgroup waits for tile j + 1 of its pipe before it releases the stage of tile j (slot B's layer 1 is issued
    // before slot A's completes), so a pipe needs at least two stages -- every two-pipe plan has them (fc_chain_plan_create).

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

    if (warp == prod_warp || (kProducerWG && warp > prod_warp)) {
        // ======================= producer (kProducerWG: its whole warpgroup gives registers away, three warps of it idle) ==========
        if (kProducerWG) asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs) : "memory");
        if (warp == prod_warp && lane == 0) {
            // weight image -> smem (same bytes for every CTA; L2-resident after the first wave).  The weights were written at model
            // build, long before any kernel that may still be running ahead of this one, so they are fetched before the grid
            // dependency is resolved.
            mbar_arrive_expect_tx(&bar_w, P.w_bytes);
            for (uint32_t off = 0; off < P.w_bytes; off += 32768)
                bulk_load_1d(smem + P.off_w + off, P.w_image + off, min(32768u, P.w_bytes - off), &bar_w);
            if (!kFloatIn) {
                // kFixed: the first tile of each of the CTA's four slots is prefetched into L2 ahead of the grid-dependency wait,
                // so that the first loads after it do not wait on HBM.  A prefetch hands no data to the CTA: the loads below
                // read the images through L2, the point of coherence that every write of an earlier kernel has reached once
                // the wait returns.
                if constexpr (kFixed) {
                    for (uint32_t i = 0; i < min(my_tiles, (uint32_t)(kPipes * kSlots)); i++)
#pragma unroll
                        for (uint32_t a = 0; a < kFixedInAtoms; a++)
                            tma_prefetch_l2_2d(&tmap_in, (int32_t)(a * 128), (int32_t)((tile0 + i * tile_step) * kTileM));
                }
                // everything else this kernel reads or writes may belong to the kernel launched before it
                if (P.wait_prior_grid) asm volatile("griddepcontrol.wait;" ::: "memory");
                const uint64_t l2_policy = policy_evict_first();   // images are read exactly once
                BNM_TRACE_DECL(kTraceWriters - 1, true);
                // the pipes take turns, so each pipe's tile is at the same ring position: one position serves them all
                RingPos ring;
                uint32_t pipe = 0;
                for (uint32_t i = 0; i < my_tiles; i++) {
                    // Only lane 0 runs this loop, so the shuffle names lane 0 alone and returns its own value.  It is kept for
                    // ptxas: with the stage computed from the counters alone, ptxas (CUDA 12.9) serialises the wgmma pipeline of
                    // the fixed-shape kernel (remark C7511).
                    const uint32_t s = __shfl_sync(1u, pipe * n_st + ring.stage(), 0);
                    BNM_TRACE(TR_EMPTY_BEGIN, 0, 0);
                    if (i >= kPipes * n_st) mbar_wait_relaxed(&bar_empty[s], ring.phase() ^ 1, P.err, 5);   // past the first round
                    BNM_TRACE(TR_EMPTY_END, 0, 0);
                    mbar_arrive_expect_tx(&bar_full[s], P.stage_bytes);
                    const int32_t row = (int32_t)((tile0 + i * tile_step) * kTileM);
                    for (uint32_t a = 0; a < P.in_atoms; a++)
                        tma_load_2d_hint(smem + s * P.stage_bytes + a * 16384, &tmap_in, (int32_t)(a * 128), row, &bar_full[s], l2_policy);
                    if (++pipe == kPipes) {
                        pipe = 0;
                        ring.advance(n_st);
                    }
                }
                BNM_TRACE_END();
            }
        }
    } else if (warp < prod_warp) {
        // ======================= consumer warpgroup cw = 2 pipe + half =======================
        if (kProducerWG) asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs) : "memory");
        const uint32_t cw = warp >> 2, pipe = cw >> 1, half = cw & 1, wq = warp & 3;
        const uint32_t quad = lane & 3;
        const uint32_t row_in_tile = half * 64 + wq * 16 + (lane >> 2);   // this thread's first row; the second is 8 below
        const int n_layers = kFixed ? kFixedLayers : P.n_layers;
        const uint32_t ncls = P.n_classes;
        // labels-only launches pass no logits buffer.  The shuffle is a value no-op (a uniform flag), kept for ptxas: testing
        // P.logits at the store instead serialises the fixed-shape kernel's wgmma pipeline (C7511, CUDA 12.9).
        const bool has_logits = __shfl_sync(0xffffffffu, (uint32_t)(kRule == kRuleEmul ? P.emul_logits != nullptr : P.logits != nullptr), 0);
        mbar_wait(&bar_w, 0, P.err, 6);   // weight tiles are in shared memory
        // B descriptor of the 64 columns from c0 of the K-step tile at smem address t (no-swizzle K-major: 8-row groups 256 B apart).
        // Every wgmma is issued at the kernel's full width kN, with no condition around it (a conditional wgmma cannot stay in
        // the asynchronous pipeline): columns past a layer's n_pad and K-steps past its k_steps read the zero tile at w_zero
        // instead (a piece that straddles n_pad reads up to 48 rows past its tile, which the zero tile behind the image also
        // covers); the epilogue ignores those columns.  With kLastN = 16 the last layer is issued 16 wide.
        const uint32_t w_zero = w_base + P.zero_off;
        auto b_desc = [](uint32_t t, int c0) { return make_smem_desc(t + (uint32_t)c0 / 8 * 256, 128, 256, GMMA_LAYOUT_NONE); };
        uint32_t acc[kSlots][kN / 2];
        uint32_t afr[kSlots][kN / 8];          // next layer's A fragments: 4 registers per K-step of 32
        BNM_TRACE_DECL(cw, wq == 0 && lane == 0);
        // kFixed: descriptors of stage 0 of this warpgroup's rows and of the weight image; every MMA adds a compile-time offset
        // (and the stage's) to them.  No layer of the class has padded K-steps or columns, so the zero tile is never read.
        const uint64_t a_base = make_smem_desc(smem_base + half * 8192, 16, 1024, GMMA_LAYOUT_SW128);
        const uint64_t w_desc = b_desc(w_base, 0);

        // ---- layer 1 into a (A: the SW128 image in stage s, this warpgroup's 64 rows start 8 KB in for the lower half)
        auto issue_layer1 = [&](uint32_t *a, uint32_t s) {
            if constexpr (kFixed) {
                const uint32_t a_s = s * (kFixedInAtoms * 16384 / 16);
                BNM_TRACE(TR_ISSUE, 0, 0);
                wgmma_fence();
#pragma unroll
                for (uint32_t k = 0; k < fixed_k_steps(0); k++)
                    wgmma_ss_n64(a, desc_add(a_base, a_s + (k >> 2) * 1024 + (k & 3) * 2), desc_add(w_desc, k * fixed_n_pad(0) * 32 / 16), k != 0);
                return;
            }
            const uint64_t a0 = make_smem_desc(smem_base + s * P.stage_bytes + half * 8192, 16, 1024, GMMA_LAYOUT_SW128);
            const uint32_t n_pad = P.n_pad[0], k_steps = P.k_steps[0];
            BNM_TRACE(TR_ISSUE, 0, 0);
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
                        wgmma_ss_n64(a + c0 / 2, ad, b_desc((uint32_t)c0 < n_pad ? bt : w_zero, c0), (pl | k) != 0);
                }
        };
        // ---- ReLUNorm of layer l's accumulators a into the A fragments f of layer l + 1, by the emulator's rule when emul is
        // std::true_type, else by the C engine's
        auto relunorm_rule = [&](const uint32_t *a, uint32_t *f, int l, auto emul) {
            // kFixed: every layer with a ReLUNorm (all but the last) is 64 wide, so every block is taken, with no predicates
            const uint32_t n_pad = kFixed ? fixed_n_pad(0) : P.n_pad[l];
            int m0 = 0, m1 = 0;
#pragma unroll
            for (int j = 0; j < kN / 8; j += 2)
                if ((uint32_t)j * 8 < n_pad) {
                    m0 = __vimax3_s32(m0, (int)a[4 * j], (int)a[4 * j + 1]);
                    m1 = __vimax3_s32(m1, (int)a[4 * j + 2], (int)a[4 * j + 3]);
                    m0 = __vimax3_s32(m0, (int)a[4 * j + 4], (int)a[4 * j + 5]);
                    m1 = __vimax3_s32(m1, (int)a[4 * j + 6], (int)a[4 * j + 7]);
                }
            m0 = max(m0, __shfl_xor_sync(0xffffffffu, m0, 1));
            m1 = max(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
            m0 = max(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
            m1 = max(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
            auto coef = [](int m) { if constexpr (decltype(emul)::value) return emul_coef(m); else return norm_coef(m); };
            const auto k0 = coef(m0), k1 = coef(m1);
            // 16-column block b -> register 2b (upper row) / 2b + 1 (lower row) of the fragments, i.e. for K-step s = b / 2:
            // f[4s] (upper row, block 2s), f[4s + 1] (lower, 2s), f[4s + 2] (upper, 2s + 1), f[4s + 3] (lower, 2s + 1)
#pragma unroll
            for (int b = 0; b < kN / 16; b++) {
                const int fi = 4 * (b >> 1) + 2 * (b & 1);
                if ((uint32_t)b * 16 < n_pad) {
                    f[fi] = norm_pack4(a[8 * b], a[8 * b + 1], a[8 * b + 4], a[8 * b + 5], k0);
                    f[fi + 1] = norm_pack4(a[8 * b + 2], a[8 * b + 3], a[8 * b + 6], a[8 * b + 7], k1);
                } else {
                    f[fi] = 0;
                    f[fi + 1] = 0;
                }
            }
        };
        auto relunorm = [&](const uint32_t *a, uint32_t *f, int l) { relunorm_rule(a, f, l, std::bool_constant<kRule == kRuleEmul>{}); };
        // ---- layer l >= 1 into a (A: the fragments f)
        auto issue_layer = [&](uint32_t *a, const uint32_t *f, int l) {
            if constexpr (kFixed) {
                // layers 2 .. 4 take 2 K-steps each, and the 64-wide layers 2 and 3 are of equal size in the weight image
                static_assert(fixed_b_off(3) == fixed_b_off(1) + 2 * fixed_k_steps(1) * fixed_n_pad(1) * 32, "kFixed weight image");
                const uint32_t b_l = (fixed_b_off(1) + (uint32_t)(l - 1) * fixed_k_steps(1) * fixed_n_pad(1) * 32) / 16;
                BNM_TRACE(TR_ISSUE, 0, l);
                wgmma_fence();
                if (l + 1 == kFixedLayers) {
#pragma unroll
                    for (uint32_t k = 0; k < fixed_k_steps(1); k++)
                        wgmma_rs_n16(a, f + 4 * k, desc_add(w_desc, b_l + k * fixed_n_pad(kFixedLayers - 1) * 32 / 16), k != 0);
                } else {
#pragma unroll
                    for (uint32_t k = 0; k < fixed_k_steps(1); k++)
                        wgmma_rs_n64(a, f + 4 * k, desc_add(w_desc, b_l + k * fixed_n_pad(1) * 32 / 16), k != 0);
                }
                return;
            }
            const uint32_t n_pad = P.n_pad[l], k_steps = P.k_steps[l], b_l = w_base + P.b_off[l];
            BNM_TRACE(TR_ISSUE, 0, l);
            wgmma_fence();
            if (kLastN < kN && l + 1 == n_layers) {
#pragma unroll 1
                for (uint32_t pl = 0; pl < P.planes[l]; pl++)
#pragma unroll
                    for (int k = 0; k < kN / 32; k++)
                        wgmma_rs_n16(a, f + 4 * k, b_desc((uint32_t)k < k_steps ? b_l + (pl * k_steps + k) * n_pad * 32 : w_zero, 0), (pl | k) != 0);
                return;
            }
#pragma unroll 1
            for (uint32_t pl = 0; pl < P.planes[l]; pl++)
#pragma unroll
                for (int k = 0; k < kN / 32; k++) {   // unrolled: the fragment index stays a compile-time constant
                    const uint32_t bt = (uint32_t)k < k_steps ? b_l + (pl * k_steps + k) * n_pad * 32 : w_zero;
#pragma unroll
                    for (int c0 = 0; c0 < kN; c0 += 64)
                        wgmma_rs_n64(a + c0 / 2, f + 4 * k, b_desc((uint32_t)c0 < n_pad ? bt : w_zero, c0), (pl | k) != 0);
                }
        };
        // ---- kOutTopK: the k best classes of tile i and their scores from the last layer's accumulators a, in place of the epilogue
        // below.  k rounds of its argmax: round 0 is that argmax; round t > 0 takes the first maximum of the columns ranked after
        // round t - 1's pick (v, p) -- x < v, or x == v at a column >= q = p + 1.  So the picks are the row's classes by logit,
        // highest first, ties to the lower class (np.argsort(-x, kind="stable")), with no exclusion mask: (v, q) per row is all the
        // state.  Rounds t > 0 start from INT32_MIN, below every logit (|logit| <= 1024 x 127 x 255 < 2^25).  Quad lane t % 4
        // keeps round t's pick; after every fourth round and after the last, the quad stores its picks: up to four consecutive
        // classes (and scores) of the row, 16 contiguous bytes.
        auto topk_epilogue = [&](const uint32_t *a, uint32_t i) {
            const uint32_t tile = tile0 + i * tile_step;
            const uint32_t k = P.k;
#pragma unroll
            for (int r = 0; r < 2; r++) {
                const size_t img = (size_t)tile * kTileM + row_in_tile + 8 * r;
                int v = INT32_MAX;
                uint32_t q = 0;
                uint32_t my_cls = 0;
                int my_score = 0;
#pragma unroll 1
                for (uint32_t t = 0; t < k; t++) {
                    int best = t ? INT32_MIN : -INT32_MAX;
                    uint32_t pos = 255;
#pragma unroll
                    for (int j = 0; j < kLastN / 8; j++)
#pragma unroll
                        for (int e = 0; e < 2; e++) {
                            const uint32_t col = 8 * j + 2 * quad + e;
                            const int x = (int)a[4 * j + 2 * r + e];
                            if (col < ncls && (x < v || (x == v && col >= q)) && x > best) { best = x; pos = col; }
                        }
#pragma unroll
                    for (int sh = 1; sh <= 2; sh <<= 1) {
                        const int ob = __shfl_xor_sync(0xffffffffu, best, sh);
                        const uint32_t op = __shfl_xor_sync(0xffffffffu, pos, sh);
                        if (ob > best || (ob == best && op < pos)) { best = ob; pos = op; }
                    }
                    v = best;
                    q = pos + 1;
                    if (quad == (t & 3)) { my_cls = pos; my_score = best; }
                    if (((t & 3) == 3 || t + 1 == k) && img < P.n && quad <= (t & 3)) {
                        const size_t o = img * k + (t & ~3u) + quad;
                        P.classes[o] = my_cls;
                        if constexpr (kRule == kRuleEmul) {
                            if (P.scores_f64) P.scores_f64[o] = (double)my_score * P.emul_logit_scale;   // exact, as the logits
                        } else {
                            if (P.scores_i32) P.scores_i32[o] = my_score;
                        }
                    }
                }
            }
        };
        // ---- logits + label of tile i from the last layer's accumulators a (dll.c:115-116: the last ReLUNorm's argmax is what
        // Inference() returns).  argmax = first maximum (strict '>' from -INT32_MAX, pos 255, inference.c:32-37): in column order
        // per thread, then over the quad.  The last layer has at most kLastN columns.
        // (row_label below is the same argmax for the two-engine kernel; the epilogue keeps its own copy, whose instruction
        // schedule in the other kernels a shared lambda would change.)
        auto epilogue = [&](const uint32_t *a, uint32_t i) {
            const uint32_t tile = tile0 + i * tile_step;
#pragma unroll
            for (int r = 0; r < 2; r++) {
                const size_t img = (size_t)tile * kTileM + row_in_tile + 8 * r;
                int best = -INT32_MAX;
                uint32_t pos = 255;
#pragma unroll
                for (int j = 0; j < kLastN / 8; j++)
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        const uint32_t col = 8 * j + 2 * quad + e;
                        const int x = (int)a[4 * j + 2 * r + e];
                        if (col < ncls && x > best) { best = x; pos = col; }
                    }
#pragma unroll
                for (int sh = 1; sh <= 2; sh <<= 1) {
                    const int ob = __shfl_xor_sync(0xffffffffu, best, sh);
                    const uint32_t op = __shfl_xor_sync(0xffffffffu, pos, sh);
                    if (ob > best || (ob == best && op < pos)) { best = ob; pos = op; }
                }
                if (kRule == kRuleEmul && img < P.n) {
                    // float64 logits: (double)acc x 2^-level_shift is exact, and argmax of the int32 accumulators is that of them
                    if (has_logits) {
                        double *d = P.emul_logits + img * ncls;
                        const double sc = P.emul_logit_scale;
#pragma unroll
                        for (int j = 0; j < kLastN / 8; j++) {
                            const uint32_t col = 8 * j + 2 * quad;
                            if (col < ncls) d[col] = (double)(int)a[4 * j + 2 * r] * sc;
                            if (col + 1 < ncls) d[col + 1] = (double)(int)a[4 * j + 2 * r + 1] * sc;
                        }
                    }
                    if (quad == 0 && P.labels) P.labels[img] = pos;
                } else if (img < P.n) {
                    auto store_row = [&](int32_t *d) {
#pragma unroll
                        for (int j = 0; j < kLastN / 8; j++) {
                            const uint32_t col = 8 * j + 2 * quad;
                            if ((ncls & 1) == 0) {   // rows are 8-byte aligned: 64-bit stores
                                if (col < ncls) *reinterpret_cast<int2 *>(d + col) = make_int2((int)a[4 * j + 2 * r], (int)a[4 * j + 2 * r + 1]);
                            } else {
                                if (col < ncls) d[col] = (int)a[4 * j + 2 * r];
                                if (col + 1 < ncls) d[col + 1] = (int)a[4 * j + 2 * r + 1];
                            }
                        }
                    };
                    if (has_logits) store_row(P.logits + img * ncls);
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
        };
        auto wait_full = [&](uint32_t s, uint32_t parity, int slot) {   // the tile of ring phase `parity` has landed in stage s
            BNM_TRACE(TR_FULL_BEGIN, slot, 0);
            mbar_wait(&bar_full[s], parity, P.err, 2);
            BNM_TRACE(TR_FULL_END, slot, 0);
        };
        auto release_stage = [&](uint32_t s) {   // this warp's reads of stage s are complete
            __syncwarp();
            if (lane == 0) mbar_arrive(&bar_empty[s]);
        };

        RingPos ring;   // ring position of the pipe's next tile
        if constexpr (kOut == kOutEngines) {
            // Both engines scale the image alike and multiply it by the same weights (the emulator's level scale cancels, see
            // emul_coef), so their layer-1 accumulators are the same: layer 1 runs once and feeds both hidden-layer rules, the
            // emulator's fragments in afr_py.  Then the C chain and the emulator's chain run one after the other from their own
            // fragments.  A one-layer model has no hidden layer: both labels are the argmax of layer 1.
            uint32_t afr_py[kN / 8];
            EngineTally tally;
            auto row_label = [&](const uint32_t *a, int r) {   // the epilogue's argmax of row r (0: this thread's first row, 1: 8 below)
                int best = -INT32_MAX;
                uint32_t pos = 255;
#pragma unroll
                for (int j = 0; j < kLastN / 8; j++)
#pragma unroll
                    for (int e = 0; e < 2; e++) {
                        const uint32_t col = 8 * j + 2 * quad + e;
                        const int x = (int)a[4 * j + 2 * r + e];
                        if (col < ncls && x > best) { best = x; pos = col; }
                    }
#pragma unroll
                for (int sh = 1; sh <= 2; sh <<= 1) {
                    const int ob = __shfl_xor_sync(0xffffffffu, best, sh);
                    const uint32_t op = __shfl_xor_sync(0xffffffffu, pos, sh);
                    if (ob > best || (ob == best && op < pos)) { best = ob; pos = op; }
                }
                return pos;
            };
#pragma unroll 1
            for (uint32_t i = 0; i < my_tiles; i++) {
                const uint32_t s = ring.stage();
                wait_full(s, ring.phase(), 0);
                ring.advance(n_st);
                issue_layer1(acc[0], s);
                wgmma_commit();
                wgmma_wait<0>();
                release_stage(s);
                uint32_t lab_c[2], lab_py[2];
                if (n_layers > 1) relunorm_rule(acc[0], afr_py, 0, std::true_type{});
                for (int l = 0;; l++) {   // the C engine
                    if (l + 1 < n_layers) {
                        relunorm_rule(acc[0], afr[0], l, std::false_type{});
                        issue_layer(acc[0], afr[0], l + 1);
                        wgmma_commit();
                        wgmma_wait<0>();
                        continue;
                    }
                    lab_c[0] = row_label(acc[0], 0);
                    lab_c[1] = row_label(acc[0], 1);
                    break;
                }
                lab_py[0] = lab_c[0];
                lab_py[1] = lab_c[1];
                for (int l = 1; l < n_layers; l++) {   // the emulator
                    issue_layer(acc[0], afr_py, l);
                    wgmma_commit();
                    wgmma_wait<0>();
                    if (l + 1 < n_layers) {
                        relunorm_rule(acc[0], afr_py, l, std::true_type{});
                    } else {
                        lab_py[0] = row_label(acc[0], 0);
                        lab_py[1] = row_label(acc[0], 1);
                    }
                }
                const size_t img0 = (size_t)(tile0 + i * tile_step) * kTileM + row_in_tile;
#pragma unroll
                for (int r = 0; r < 2; r++) {
                    const size_t img = img0 + 8 * r;
                    const bool row = quad == 0 && img < P.n;
                    uint32_t truth = ~0u;
                    if (row) {
                        if (P.labels) P.labels[img] = lab_c[r];
                        if (P.labels_py) P.labels_py[img] = lab_py[r];
                        if (P.truth) truth = P.truth[img];
                    }
                    tally.add(row, lab_c[r], lab_py[r], truth, ncls);
                }
            }
            if (P.counts) {
                tally.flush(P.counts);
                if (blockIdx.x == 0 && tid == 0) atomicAdd(&P.counts[0], (unsigned long long)P.n);
            }
        } else if constexpr (kSlots == 1) {
            // one tile at a time: every layer's MMAs complete before its ReLUNorm starts.  (The slot loop below would serve one
            // slot as well, but ptxas gives it about 10 to 20 more registers per one-slot instantiation and spills at kN = 256.)
#pragma unroll 1
            for (uint32_t i = pipe; i < my_tiles; i += kPipes) {
                const uint32_t s = pipe * n_st + ring.stage();
                wait_full(s, ring.phase(), 0);
                ring.advance(n_st);
                issue_layer1(acc[0], s);
                wgmma_commit();
                BNM_TRACE(TR_WAIT_BEGIN, 0, 0);
                wgmma_wait<0>();
                BNM_TRACE(TR_WAIT_END, 0, 0);
                release_stage(s);
                for (int l = 0;; l++) {
                    if (l + 1 < n_layers) {
                        relunorm(acc[0], afr[0], l);
                        issue_layer(acc[0], afr[0], l + 1);
                        wgmma_commit();
                        BNM_TRACE(TR_WAIT_BEGIN, 0, l + 1);
                        wgmma_wait<0>();
                        BNM_TRACE(TR_WAIT_END, 0, l + 1);
                        continue;
                    }
                    if constexpr (kOut == kOutTopK) topk_epilogue(acc[0], i);
                    else epilogue(acc[0], i);
                    BNM_TRACE(TR_EPI_END, 0, 0);
                    break;
                }
            }
        } else {
            // two slots, stepped alternately.  Each step of slot x commits exactly one wgmma group (empty once x has no tile left),
            // so the older of the two groups in flight is always x's and wait_group 1 means "x's MMAs are complete".  A step then
            // runs x's ReLUNorm and issues its next layer, or, after the last layer, x's epilogue and the layer 1 of the pipe's
            // next tile -- all while the other slot's group is in flight.
            uint32_t ti[kSlots];   // tile of slot x (>= my_tiles: none left)
            int ly[kSlots];        // its layer in flight
            uint32_t st[kSlots], ph[kSlots];   // its stage and ring phase
            uint32_t next = pipe;  // next tile of this pipe to take
            auto take_tile = [&](int x) {   // slot x takes the pipe's next tile and, if there is one, issues its layer 1
                ti[x] = next;
                ly[x] = 0;
                next += kPipes;
                st[x] = pipe * n_st + ring.stage();
                ph[x] = ring.phase();
                ring.advance(n_st);
                if (ti[x] < my_tiles) {
                    wait_full(st[x], ph[x], x);
                    issue_layer1(acc[x], st[x]);
                }
            };
#pragma unroll
            for (int x = 0; x < kSlots; x++) {
                take_tile(x);
                wgmma_commit();
            }
#pragma unroll 1
            while (ti[0] < my_tiles || ti[1] < my_tiles) {
#pragma unroll
                for (int x = 0; x < kSlots; x++) {
                    BNM_TRACE(TR_WAIT_BEGIN, x, ly[x]);
                    wgmma_wait<kSlots - 1>();
                    BNM_TRACE(TR_WAIT_END, x, ly[x]);
                    if (ti[x] < my_tiles) {
                        if (ly[x] == 0) release_stage(st[x]);
                        if (ly[x] + 1 < n_layers) {
                            relunorm(acc[x], afr[x], ly[x]);
                            ly[x]++;
                            issue_layer(acc[x], afr[x], ly[x]);
                        } else {
                            epilogue(acc[x], ti[x]);
                            BNM_TRACE(TR_EPI_END, x, 0);
                            take_tile(x);
                        }
                    }
                    wgmma_commit();
                }
            }
            wgmma_wait<0>();
        }
        BNM_TRACE_END();
        BNM_TRACE_STAMP(1);
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
        RingPos pos;           // ring position of the current tile (one pipe)
        if (n_groups > 0) issue_group(0);
        if (n_groups > 1) issue_group(1);
        for (uint32_t gi = 0; gi < n_groups; gi++) {
            const uint32_t i = gi / kGroupsPerTile, k = gi % kGroupsPerTile;
            const uint32_t s = pos.stage();
            if (k == 0 && i >= n_st) mbar_wait(&bar_empty[s], pos.phase() ^ 1, P.err, 8);   // the tile that used this stage is through layer 1
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
                pos.advance(n_st);
            }
        }
    }
}

template <int kN, int kPipes, bool kFloatIn, int kSlots = 1, int kLastN = kN, bool kFixed = false>
__global__ void __launch_bounds__(chain_threads<kN, kPipes, kFloatIn, kSlots>(), 1)
fc_chain_kernel(const __grid_constant__ CUtensorMap tmap_in, const __grid_constant__ ChainParams P) {
    fc_chain_body<kN, kPipes, kFloatIn, kSlots, kLastN, kFixed, kRuleC, kOutLogits>(tmap_in, P);
}

// QuantizedModel.inference_quantized (BitNetMCU.py:420-535) of FC models: the float-input launch <64,1,float> with the emulator's
// hidden-layer rule and float64 logits.  The input scaling of BitNetMCU.py:435-436 is the quantiser warps' (test_inference.py:140-141).
__global__ void __launch_bounds__(chain_threads<64, 1, true, 1>(), 1)
fc_emul_kernel(const __grid_constant__ CUtensorMap tmap_in, const __grid_constant__ ChainParams P) {
    fc_chain_body<64, 1, true, 1, 64, false, kRuleEmul, kOutLogits>(tmap_in, P);
}

// The same emulator on int8 rows that are already scaled (k_quantize_images, or the features of k_cnn_emul_frontend): TMA
// loads, one pipe, one slot, the last layer at the full width kN -- every width, and up to kN classes.
template <int kN>
__global__ void __launch_bounds__(chain_threads<kN, 1, false, 1>(), 1)
fc_emul_i8_kernel(const __grid_constant__ CUtensorMap tmap_in, const __grid_constant__ ChainParams P) {
    fc_chain_body<kN, 1, false, 1, kN, false, kRuleEmul, kOutLogits>(tmap_in, P);
}

// The reference's check of its two engines (test_inference.py:130-175) in one pass: the float-input launch <64,1,float> that
// runs the C engine's chain and the emulator's after one shared layer 1, and writes both labels and their counts.
__global__ void __launch_bounds__(chain_threads<64, 1, true, 1>(), 1)
fc_engines_kernel(const __grid_constant__ CUtensorMap tmap_in, const __grid_constant__ ChainParams P) {
    fc_chain_body<64, 1, true, 1, 64, false, kRuleBoth, kOutEngines>(tmap_in, P);
}

// Top-k on int8 rows: the chain of fc_chain_kernel (kEmul false) or of fc_emul_i8_kernel (true) on one pipe and one slot at the
// full width kN, with an epilogue that writes the k best classes of every row and their scores instead of logits and label.
template <int kN, bool kEmul>
__global__ void __launch_bounds__(chain_threads<kN, 1, false, 1>(), 1)
fc_topk_kernel(const __grid_constant__ CUtensorMap tmap_in, const __grid_constant__ ChainParams P) {
    fc_chain_body<kN, 1, false, 1, kN, false, kEmul ? kRuleEmul : kRuleC, kOutTopK>(tmap_in, P);
}

// ---------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode_fn() {
    static const EncodeTiledFn fn = [] {   // initialised once, whichever thread creates the first plan
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            return (EncodeTiledFn)p;
        return (EncodeTiledFn)nullptr;
    }();
    return fn;
}

static uint32_t round_up(uint32_t v, uint32_t m) { return (v + m - 1) / m * m; }

#ifdef BNM_FC_TRACE
// diagnostics build: with BNM_FC_TRACE_OUT set, every launch clears the trace buffer first and writes it to that file after the
// kernel has completed (the layout of FcTrace, preceded by kTraceCtas, kTraceWriters, kTraceEvents as three uint32)
static void trace_before(cudaStream_t st) {
    void *d = nullptr;
    if (getenv("BNM_FC_TRACE_OUT") && cudaGetSymbolAddress(&d, g_fc_trace) == cudaSuccess) cudaMemsetAsync(d, 0, sizeof(FcTrace), st);
}
static void trace_after(cudaStream_t st) {
    const char *path = getenv("BNM_FC_TRACE_OUT");
    if (!path || cudaStreamSynchronize(st) != cudaSuccess) return;
    std::vector<uint8_t> buf(sizeof(FcTrace));
    if (cudaMemcpyFromSymbol(buf.data(), g_fc_trace, sizeof(FcTrace)) != cudaSuccess) return;
    if (FILE *f = fopen(path, "wb")) {
        const uint32_t dims[3] = {kTraceCtas, kTraceWriters, kTraceEvents};
        fwrite(dims, sizeof(dims), 1, f);
        fwrite(buf.data(), buf.size(), 1, f);
        fclose(f);
    }
}
#else
static void trace_before(cudaStream_t) {}
static void trace_after(cudaStream_t) {}
#endif

// a kernel row: one __global__ instantiation, named by its function and its template arguments <kN, kPipes, kSlots, kLastN>
struct ChainKernel {
    const char *name;
    void (*fn)(CUtensorMap, ChainParams);
    int threads;
};
template <int kN, int kPipes = 1, bool kFloatIn = false, int kSlots = 1>
static constexpr ChainKernel row(const char *name, void (*fn)(CUtensorMap, ChainParams)) {
    return {name, fn, chain_threads<kN, kPipes, kFloatIn, kSlots>()};
}

// The launch forms, indexed by FcForm.  A launch takes everything but its buffers from its form's entry.
struct FormSpec {
    bool float_in;           // float32 rows through the quantiser warps, else int8 rows over TMA
    FcRule rule;
    FcOut out;               // kOutLogits: the C engine on int8 rows alone also takes result-exchange destinations
    uint32_t stage_cap;      // stages per pipe at most
    ChainKernel rows[4];     // by accumulator width 64, 128, 192, 256; fn null: the form has no row at that width
};
// The float-input forms have a 64-wide row only: the eight quantiser warps make 17 warps, so at most 96 registers per thread.
static const FormSpec kForms[kFcForms] = {
    // kFormInt8; a 64-wide plan with room for two pipes takes one of kTwoPipeRows instead of the one-pipe row
    {false, kRuleC, kOutLogits, 6,
     {row<64>("fc_chain_kernel<64,1>", fc_chain_kernel<64, 1, false>), row<128>("fc_chain_kernel<128,1>", fc_chain_kernel<128, 1, false>),
      row<192>("fc_chain_kernel<192,1>", fc_chain_kernel<192, 1, false>), row<256>("fc_chain_kernel<256,1>", fc_chain_kernel<256, 1, false>)}},
    // kFormFloat
    {true, kRuleC, kOutLogits, 4, {row<64, 1, true>("fc_chain_kernel<64,1,float>", fc_chain_kernel<64, 1, true>)}},
    // kFormEmulFloat
    {true, kRuleEmul, kOutLogits, 4, {row<64, 1, true>("fc_emul_kernel<64,1,float,emul>", fc_emul_kernel)}},
    // kFormEmulInt8
    {false, kRuleEmul, kOutLogits, 6,
     {row<64>("fc_emul_i8_kernel<64,1,emul>", fc_emul_i8_kernel<64>), row<128>("fc_emul_i8_kernel<128,1,emul>", fc_emul_i8_kernel<128>),
      row<192>("fc_emul_i8_kernel<192,1,emul>", fc_emul_i8_kernel<192>), row<256>("fc_emul_i8_kernel<256,1,emul>", fc_emul_i8_kernel<256>)}},
    // kFormEngines
    {true, kRuleBoth, kOutEngines, 4, {row<64, 1, true>("fc_engines_kernel<64,1,float,engines>", fc_engines_kernel)}},
    // kFormTopK
    {false, kRuleC, kOutTopK, 6,
     {row<64>("fc_topk_kernel<64,1,topk>", fc_topk_kernel<64, false>), row<128>("fc_topk_kernel<128,1,topk>", fc_topk_kernel<128, false>),
      row<192>("fc_topk_kernel<192,1,topk>", fc_topk_kernel<192, false>), row<256>("fc_topk_kernel<256,1,topk>", fc_topk_kernel<256, false>)}},
    // kFormEmulTopK
    {false, kRuleEmul, kOutTopK, 6,
     {row<64>("fc_topk_kernel<64,1,emul,topk>", fc_topk_kernel<64, true>), row<128>("fc_topk_kernel<128,1,emul,topk>", fc_topk_kernel<128, true>),
      row<192>("fc_topk_kernel<192,1,emul,topk>", fc_topk_kernel<192, true>), row<256>("fc_topk_kernel<256,1,emul,topk>", fc_topk_kernel<256, true>)}},
};
// kFormInt8's two-pipe two-slot rows: the last layer at full width, 16 wide (kLastN, for heads of at most 16 classes), or the
// fixed-shape kernel
static const ChainKernel kTwoPipeRows[3] = {
    row<64, 2, false, 2>("fc_chain_kernel<64,2,2,64>", fc_chain_kernel<64, 2, false, 2>),
    row<64, 2, false, 2>("fc_chain_kernel<64,2,2,16>", fc_chain_kernel<64, 2, false, 2, 16>),
    row<64, 2, false, 2>("fc_chain_kernel<64,2,2,16,fixed>", fc_chain_kernel<64, 2, false, 2, 16, true>),
};

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
    max_n = round_up(max_n, 64);
    p.zero_off = w_off;                    // [max_n x 32 B] of zeros behind the layers (cudaMemset below)
    p.w_bytes = w_off + max_n * 32;
    p.n_classes = layers[n_layers - 1].n_out;
    p.emul_logit_scale = level_shift_of(layers[n_layers - 1].enc) ? 0.5 : 1.0;
    const uint32_t smem_limit = 227 * 1024 - 1024 /*alignment slack*/ - 1024 /*static: barriers*/;
    const uint32_t w_fixed = round_up(p.w_bytes, 128);
    if (w_fixed + 2 * p.stage_bytes > smem_limit) { delete plan; return fail("fused path: weights do not fit in shared memory"); }
    // the int8 C-engine form of a 64-wide model runs two pipes where four stages fit.  Two pipes run two slots, which issue a last
    // layer of at most 16 columns 16 wide (kLastN); plans of exactly the fixed shape class (kFixedLayers and the fixed_* shapes)
    // run the fixed-shape kernel
    const uint32_t pipes = (max_n == 64 && (smem_limit - w_fixed) / p.stage_bytes >= 4) ? 2 : 1;
    const bool last16 = layers[n_layers - 1].n_pad <= 16;
    bool fixed = pipes == 2 && last16 && n_layers == kFixedLayers && p.in_atoms == kFixedInAtoms;
    for (int l = 0; l < n_layers && fixed; l++)
        fixed = p.planes[l] == 1 && p.n_pad[l] == fixed_n_pad(l) && p.k_steps[l] == fixed_k_steps(l) && p.b_off[l] == fixed_b_off(l);
    // the float-input forms (one pipe, fewer int8 stages) hold the quantiser warps' float rings in the shared memory they free:
    // rows of at most 256 elements and at most 16 classes
    const uint32_t fring = kFloatQuantWarps * 2 * kFloatGroupRows * 1024;
    const bool float_fits = in_bytes <= 256 && p.n_classes <= 16 && w_fixed + fring + 2 * p.stage_bytes <= smem_limit;
    FormLayout *forms = plan->forms;
    for (int f = 0; f < kFcForms; f++) {
        const FormSpec &s = kForms[f];
        const uint32_t np = f == kFormInt8 ? pipes : 1;
        const ChainKernel *k = np == 2 ? &kTwoPipeRows[fixed ? 2 : last16 ? 1 : 0] : &s.rows[max_n / 64 - 1];
        if (!k->fn || (s.float_in && !float_fits)) continue;
        // the layout: np rings of stages in what the weight image and `extra` bytes (the float rings) leave, at most kMaxStages
        // over the pipes (>= 2 per pipe with two: two tile slots need it), then the weights, then the extra bytes
        FormLayout &l = forms[f];
        const uint32_t extra = s.float_in ? fring : 0;
        l.kernel = k;
        l.n_stages = std::min({s.stage_cap, kMaxStages / np, (smem_limit - w_fixed - extra) / p.stage_bytes / np});
        l.off_w = np * l.n_stages * p.stage_bytes;
        l.off_fring = extra ? l.off_w + w_fixed : 0;
        // One CTA per SM is part of the launch-overlap contract (launch k+2 must never run next to launch k on an SM): shared
        // memory enforces it once a CTA asks for more than half of the SM's 227 kB.
        l.smem_bytes = std::max<size_t>((size_t)l.off_w + w_fixed + extra + 1024, 116 * 1024);
    }
    if (getenv("BNM_VERBOSE")) {   // diagnostics: the shapes this plan launches
        const bool has_float = forms[kFormFloat].kernel;
        auto args = [&](FcForm f) { return has_float ? strchr(forms[f].kernel->name, '<') : ""; };   // the template arguments
        char f_stages[32] = "";
        if (has_float) snprintf(f_stages, sizeof(f_stages), ", float input stages %u", forms[kFormFloat].n_stages);
        fprintf(stderr, "bitnetmcu_b200: fused FC plan: %u accumulator columns, %u pipes x %u stages, %u weight bytes, %zu B smem, "
                "%s%s%s%s%s%s, int8 emulator %s x %u stages\n", max_n, pipes, forms[kFormInt8].n_stages, p.w_bytes,
                forms[kFormInt8].smem_bytes, forms[kFormInt8].kernel->name, has_float ? ", float input " : "", args(kFormFloat),
                has_float ? ", emulator " : "", args(kFormEmulFloat), f_stages, forms[kFormEmulInt8].kernel->name,
                forms[kFormEmulInt8].n_stages);
        fprintf(stderr, "bitnetmcu_b200: fused FC top-k forms: %s x %u stages, emulator %s x %u stages, %zu B smem\n",
                forms[kFormTopK].kernel->name, forms[kFormTopK].n_stages, forms[kFormEmulTopK].kernel->name, forms[kFormEmulTopK].n_stages,
                forms[kFormTopK].smem_bytes);
    }
    plan->verbose = getenv("BNM_VERBOSE") != nullptr;
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
    for (const FormLayout &f : plan->forms)
        if (f.kernel && !raise_smem_limit((const void *)f.kernel->fn, f.smem_bytes)) {
            fc_chain_plan_destroy(plan);
            return fail("cannot opt in to the required dynamic shared memory");
        }
    return plan;
}

void fc_chain_plan_set_overlap(FcChainPlan *p, int mode) {
    if (!p) return;
    std::lock_guard<std::mutex> lock(p->mu);
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

bool fc_chain_has_form(const FcChainPlan *plan, FcForm f) { return plan && plan->forms[f].kernel; }

const char *fc_chain_form_name(const FcChainPlan *plan, FcForm f) { return plan->forms[f].kernel->name; }

static const CUtensorMap kNoTensorMap{};   // the float-input forms' tensor map: not used (no TMA image loads)

int fc_chain_launch(FcChainPlan *plan, FcForm f, const void *in, size_t n, const FcOutputs &out, cudaStream_t st) {
    if (n == 0) return 0;
    if (n > 0x7fffff00ull) return -2;
    const FormLayout &form = plan->forms[f];
    if (!form.kernel) return -6;
    const FormSpec &s = kForms[f];
    // the C engine on int8 rows: the one form with result-exchange destinations and overlapping launches
    const bool engine_i8 = !s.float_in && s.rule == kRuleC && s.out == kOutLogits;
    const EngineOutputs &e = out.engines;
    const TopKOutputs &t = out.topk;
    if ((out.logits && s.out != kOutLogits) || (out.gather && !engine_i8) || ((e.labels_py || e.truth || e.counts) && s.out != kOutEngines) ||
        (s.out == kOutTopK) != (t.k != 0) || (t.k && (out.labels || !t.classes || t.k > plan->p.n_classes)))
        return -5;
    ChainParams p = plan->p;   // the model's shapes and the emulator's logit scale; null outputs, no result exchange
    p.n_stages = form.n_stages;
    p.off_w = form.off_w;
    p.off_fring = form.off_fring;
    if (s.rule == kRuleEmul) {
        p.emul_logits = static_cast<double *>(out.logits);
        p.scores_f64 = static_cast<double *>(t.scores);
    } else {
        p.logits = static_cast<int32_t *>(out.logits);
        p.scores_i32 = static_cast<int32_t *>(t.scores);
    }
    p.labels = out.labels;
    p.labels_py = e.labels_py;
    p.truth = e.truth;
    p.counts = e.counts;
    p.k = t.k;
    p.classes = t.classes;
    p.n = n;
    p.n_tiles = (uint32_t)((n + kTileM - 1) / kTileM);
    if (const GatherDst *gather = out.gather) {
        if (gather->n_labels_dst > (uint32_t)kMaxGatherDst || gather->n_logits_dst > (uint32_t)kMaxGatherDst) return -5;
        p.n_lab_dst = gather->n_labels_dst;
        p.n_log_dst = gather->n_logits_dst;
        p.row0 = gather->row_offset;
        p.lab_u8 = gather->labels_u8 && p.n_classes <= 255;
        if (gather->labels_u8 && !p.lab_u8) return -5;
        for (uint32_t d = 0; d < p.n_lab_dst; d++) p.lab_dst[d] = gather->labels_dst[d];
        for (uint32_t d = 0; d < p.n_log_dst; d++) p.log_dst[d] = gather->logits_dst[d];
    }
    // From the tensor-map lookup to the launch, one thread at a time per plan: the cached map must not be rewritten before the
    // launch has copied it, and "the previous launch" of mode 2 is the previous launch enqueued on this plan, from any thread.
    std::lock_guard<std::mutex> lock(plan->mu);
    const CUtensorMap *tmap_p = &kNoTensorMap;
    if (s.float_in) {
        p.fimages = static_cast<const float *>(in);
        p.in_elems = plan->in_bytes;
    } else if (!(tmap_p = plan_tensor_map(plan, static_cast<const int8_t *>(in), n))) {
        return -3;
    }
    // a CTA per tile, at most one per SM
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3((unsigned)std::min<uint32_t>(p.n_tiles, (uint32_t)plan->sm_count));
    cfg.blockDim = dim3(form.kernel->threads);
    cfg.dynamicSmemBytes = form.smem_bytes;
    cfg.stream = st;
    // Only the C engine's int8 form overlaps launches; every other form is a plain launch, ordered by the stream alone, whose
    // grid-dependency wait returns at once.  The int8 form is always a programmatic dependent launch: modes 0 and 1 are one
    // launch, whose CTAs take each SM as the kernel before them leaves it and run their prologue (barriers, setmaxnreg, weight
    // copy) there, but read images and write results only after the grid-dependency wait -- ordinary stream semantics.
    // Mode 2 drops the wait, i.e. EVERY ordering against the work enqueued before this launch on the stream (the previous bnm
    // launch and any producer kernel of `images` alike).  The library keeps the wait whenever it can see the promise being
    // broken: first launch on this plan / another stream / a buffer of the previous launch touched again, in any role (one
    // launch's logits the next one's images, say) / a launch of another form in between.  A null output is no buffer: it
    // neither reuses nor differs from one.
    LaunchBuffers bufs;
    bufs.io[0] = in; bufs.io[1] = out.logits; bufs.io[2] = out.labels;
    if (out.gather) {
        for (uint32_t d = 0; d < p.n_lab_dst; d++) bufs.dst[bufs.n_dst++] = p.lab_dst[d];
        for (uint32_t d = 0; d < p.n_log_dst; d++) bufs.dst[bufs.n_dst++] = p.log_dst[d];
        bufs.row0 = p.row0;
    }
    const bool independent = engine_i8 && plan->overlap == 2 && plan->prev_valid && plan->prev_stream == st && !shares_buffer(plan->prev, bufs);
    p.wait_prior_grid = !independent;
    p.early_trigger = engine_i8 && cfg.gridDim.x == (unsigned)plan->sm_count;
    plan->prev = bufs; plan->prev_stream = st; plan->prev_valid = engine_i8;
    if (engine_i8 && plan->verbose) fprintf(stderr, "bitnetmcu_b200: fused launch: %s\n", independent ? "independent" : "wait");
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = engine_i8 ? 1 : 0;
    trace_before(st);
    if (cudaLaunchKernelEx(&cfg, form.kernel->fn, *tmap_p, p) != cudaSuccess) return -4;
    trace_after(st);
    return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

}  // namespace bnm
