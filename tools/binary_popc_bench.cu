// binary_popc_bench.cu -- evidence for the "XNOR/popcount vs integer MMA" choice on Binary (1-bit) layers.
//
// BASELINE.json config 3 names an "XNOR/popcount kernel path" for Binary weights.  BitNetMCU's activations are int8, not
// 1-bit (BitNetMCU_inference.c:96-108 adds or subtracts the int8 activation per weight bit), so a popcount formulation has
// to go through 8 activation bit-planes:   sum_i a_i w_i = sum_i a_i - 2 * sum_b c_b * popc(W & P_b),  c_b = 2^b (b<7), -128 (b=7).
// This tool measures one Binary layer 256 -> 160 over a batch on CUDA cores both ways and checks that they agree:
//   A. dp4a on weights pre-decoded to +-1 int8 (what BNM_PATH_LAYERS does)
//   B. bit-plane AND/POPC (planes extracted with warp ballots, the cheapest extraction there is)
// The fused tensor-core path decodes Binary weights once per model and runs them as int8 MMAs instead.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o binary_popc_bench binary_popc_bench.cu
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>

constexpr int K = 256, NOUT = 160, KW = K / 32, OPL = NOUT / 32;   // 8 weight words per output, 5 outputs per lane

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at line %d\n", cudaGetErrorString(e_), __LINE__); exit(1); } } while (0)

// A: warp per image, lane -> outputs lane, lane+32, ...; weights int8 [k/4][NOUT] words in shared memory
__global__ void __launch_bounds__(256) k_dp4a(const int8_t *__restrict__ act, const uint32_t *__restrict__ w4, int32_t *__restrict__ out, size_t n) {
    __shared__ uint32_t sw[(K / 4) * NOUT];
    for (int i = threadIdx.x; i < (K / 4) * NOUT; i += blockDim.x) sw[i] = w4[i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    for (size_t img = (size_t)blockIdx.x * 8 + (threadIdx.x >> 5); img < n; img += (size_t)gridDim.x * 8) {
        const uint32_t *a = reinterpret_cast<const uint32_t *>(act + img * K);
        int32_t acc[OPL] = {};
#pragma unroll 16
        for (int k = 0; k < K / 4; ++k) {
            const uint32_t av = __ldg(a + k);                     // same address in all lanes: one broadcast load
#pragma unroll
            for (int o = 0; o < OPL; ++o) acc[o] = __dp4a((int)av, (int)sw[k * NOUT + o * 32 + lane], acc[o]);
        }
#pragma unroll
        for (int o = 0; o < OPL; ++o) out[img * NOUT + o * 32 + lane] = acc[o];
    }
}

// B: warp per image; 8 bit-planes x 8 words by ballot, then AND/POPC against the packed weight words (bit set = -1)
__global__ void __launch_bounds__(256) k_popc(const int8_t *__restrict__ act, const uint32_t *__restrict__ wbits, int32_t *__restrict__ out, size_t n) {
    __shared__ uint32_t sw[KW * NOUT];                            // [word][output]
    for (int i = threadIdx.x; i < KW * NOUT; i += blockDim.x) sw[i] = wbits[i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    for (size_t img = (size_t)blockIdx.x * 8 + (threadIdx.x >> 5); img < n; img += (size_t)gridDim.x * 8) {
        const int8_t *a = act + img * K;
        uint32_t plane[8][KW];
        int32_t total = 0;
#pragma unroll
        for (int wd = 0; wd < KW; ++wd) {
            const int v = a[wd * 32 + lane];
            total += v;
#pragma unroll
            for (int b = 0; b < 8; ++b) plane[b][wd] = __ballot_sync(0xffffffffu, (v >> b) & 1);
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) total += __shfl_xor_sync(0xffffffffu, total, off);
#pragma unroll
        for (int o = 0; o < OPL; ++o) {
            int32_t neg = 0;                                       // sum of activations whose weight bit is set
#pragma unroll
            for (int b = 0; b < 8; ++b) {
                int32_t c = 0;
#pragma unroll
                for (int wd = 0; wd < KW; ++wd) c += __popc(plane[b][wd] & sw[wd * NOUT + o * 32 + lane]);
                neg += (b == 7) ? -128 * c : (c << b);
            }
            out[img * NOUT + o * 32 + lane] = total - 2 * neg;
        }
    }
}

int main(int argc, char **argv) {
    const size_t n = argc > 1 ? strtoull(argv[1], nullptr, 0) : (1u << 19);
    std::vector<int8_t> act(n * K);
    std::vector<uint32_t> wbits(KW * NOUT), w4((K / 4) * NOUT);
    uint32_t s = 12345;
    auto rnd = [&]() { s = s * 1664525u + 1013904223u; return s >> 8; };
    for (auto &v : act) v = (int8_t)(rnd() & 0x7f);               // post-ReLUNorm range 0..127
    for (size_t i = 0; i < 64 && i < n; ++i) for (int k = 0; k < K; ++k) act[i * K + k] = (int8_t)(rnd() & 0xff);   // and some full-range rows
    for (auto &v : wbits) v = rnd() ^ (rnd() << 12);
    for (int o = 0; o < NOUT; ++o)
        for (int k4 = 0; k4 < K / 4; ++k4) {
            uint32_t word = 0;
            for (int j = 0; j < 4; ++j) {
                const int k = k4 * 4 + j;
                const int bit = (wbits[(k / 32) * NOUT + o] >> (k % 32)) & 1;
                word |= (uint32_t)(uint8_t)(bit ? -1 : 1) << (8 * j);
            }
            w4[k4 * NOUT + o] = word;
        }
    int8_t *d_act; uint32_t *d_wb, *d_w4; int32_t *d_a, *d_b;
    CK(cudaMalloc(&d_act, act.size())); CK(cudaMalloc(&d_wb, wbits.size() * 4)); CK(cudaMalloc(&d_w4, w4.size() * 4));
    CK(cudaMalloc(&d_a, n * NOUT * 4)); CK(cudaMalloc(&d_b, n * NOUT * 4));
    CK(cudaMemcpy(d_act, act.data(), act.size(), cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_wb, wbits.data(), wbits.size() * 4, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_w4, w4.data(), w4.size() * 4, cudaMemcpyHostToDevice));
    int sms = 0; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    const int grid = sms * 8;
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    float ms_a = 0, ms_b = 0;
    for (int rep = 0; rep < 4; ++rep) {                            // first rep = warm-up
        CK(cudaEventRecord(e0)); k_dp4a<<<grid, 256>>>(d_act, d_w4, d_a, n); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
        float t; CK(cudaEventElapsedTime(&t, e0, e1)); if (rep) ms_a += t / 3;
        CK(cudaEventRecord(e0)); k_popc<<<grid, 256>>>(d_act, d_wb, d_b, n); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
        CK(cudaEventElapsedTime(&t, e0, e1)); if (rep) ms_b += t / 3;
    }
    CK(cudaGetLastError());
    std::vector<int32_t> ha(n * NOUT), hb(n * NOUT);
    CK(cudaMemcpy(ha.data(), d_a, ha.size() * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(hb.data(), d_b, hb.size() * 4, cudaMemcpyDeviceToHost));
    size_t bad = 0;
    for (size_t i = 0; i < ha.size(); ++i) bad += ha[i] != hb[i];
    // host check of a few rows
    for (size_t i = 0; i < 8 && i < n; ++i)
        for (int o = 0; o < NOUT; ++o) {
            int32_t r = 0;
            for (int k = 0; k < K; ++k) r += ((wbits[(k / 32) * NOUT + o] >> (k % 32)) & 1) ? -act[i * K + k] : act[i * K + k];
            bad += r != ha[i * NOUT + o];
        }
    const double macs = (double)n * K * NOUT;
    printf("binary layer %d->%d, %zu images, %d SMs\n", K, NOUT, n, sms);
    printf("A dp4a (+-1 int8 weights)   : %8.3f ms  %7.2f M img/s  %6.2f TMAC/s\n", ms_a, n / ms_a / 1e3, macs / ms_a / 1e9);
    printf("B bit-plane AND/POPC        : %8.3f ms  %7.2f M img/s  %6.2f TMAC/s\n", ms_b, n / ms_b / 1e3, macs / ms_b / 1e9);
    printf("mismatches A vs B vs host   : %zu\n", bad);
    return bad != 0;
}
