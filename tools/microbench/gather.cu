// tools/microbench/gather.cu -- what can one SM sustain on the head kernel's table gathers?
//
// The fused head kernel spends ~40 % of a batch in two gather phases: every thread issues EIGHT scattered 32-byte
// (one-sector) loads into a 29 MB L2-resident table, waits for all of them, and blends.  This standalone probe issues the
// same access pattern with nothing else in the way, so the phase time measured in the kernel (tools/phase_breakdown.py)
// can be compared with what the memory system gives when asked nicely.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/microbench/gather.bin tools/microbench/gather.cu
//   tools/microbench/gather.bin            # prints one line per configuration
//
// Reported per configuration: cycles per "phase" (= one round of K loads per thread, all threads of the SM), sectors per
// clock per SM, and aggregate GB/s.  Knobs: loads in flight per thread K, resident CTAs per SM (via dynamic smem, like the
// real kernel: 2 x 112 KB leaves ~28 KB of L1), L1 allocation policy, spatial locality of consecutive threads.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1); } } while (0)

__device__ __forceinline__ void ldg256(const uint4 *p, uint4 &lo, uint4 &hi, bool noalloc) {
    unsigned long long a, b, c, d;
    if (noalloc) asm volatile("ld.global.nc.L1::no_allocate.v4.u64 {%0,%1,%2,%3}, [%4];" : "=l"(a), "=l"(b), "=l"(c), "=l"(d) : "l"(p));
    else asm volatile("ld.global.nc.v4.u64 {%0,%1,%2,%3}, [%4];" : "=l"(a), "=l"(b), "=l"(c), "=l"(d) : "l"(p));
    lo.x = (uint32_t)a; lo.y = (uint32_t)(a >> 32); lo.z = (uint32_t)b; lo.w = (uint32_t)(b >> 32);
    hi.x = (uint32_t)c; hi.y = (uint32_t)(c >> 32); hi.z = (uint32_t)d; hi.w = (uint32_t)(d >> 32);
}
__device__ __forceinline__ uint32_t mix(uint32_t x) {
    x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
    return x;
}

// `spread`: neighbouring threads read entries within +-spread of a common random base (0 = fully random): samples of
// neighbouring rays land in neighbouring cells, which is where the real kernel's L1 hits come from.
template <int K>
__global__ void __launch_bounds__(256) k_gather(const uint4 *__restrict__ table, uint32_t entries, int phases, int spread, int noalloc,
                                                unsigned long long *cycles, uint32_t *sink) {
    extern __shared__ unsigned char pad_[];
    const uint32_t gtid = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t acc = 0;
    __syncthreads();
    const long long t0 = clock64();
    for (int p = 0; p < phases; ++p) {
        uint4 lo[K], hi[K];
#pragma unroll
        for (int j = 0; j < K; ++j) {
            uint32_t e;
            if (spread) {
                const uint32_t base = mix((gtid >> 5) * 977u + p * 131071u + j * 7919u) % entries;     // one base per warp
                e = (base + mix(gtid * 31u + p + j) % (uint32_t)spread) % entries;
            } else {
                e = mix(gtid * 2654435761u + p * 40503u + j * 9973u) % entries;
            }
            ldg256(table + 2 * (size_t)e, lo[j], hi[j], noalloc != 0);
        }
#pragma unroll
        for (int j = 0; j < K; ++j) acc += lo[j].x ^ lo[j].w ^ hi[j].y ^ hi[j].z;
        __syncthreads();   // the real kernel ends every gather phase with a CTA barrier
    }
    const long long t1 = clock64();
    if (threadIdx.x == 0) atomicAdd(cycles, (unsigned long long)(t1 - t0));
    if (acc == 0x12345678u) sink[0] = acc + pad_[0];
}

template <int K>
static void run(const uint4 *table, uint32_t entries, int ctas_per_sm, int spread, int noalloc, int sms, unsigned long long *d_cyc, uint32_t *d_sink) {
    const int phases = 400;
    // dynamic smem sized so that exactly `ctas_per_sm` CTAs fit, the way the head kernel's operand tiles do
    const int smem = (ctas_per_sm == 1) ? 200 * 1024 : (ctas_per_sm == 2) ? 111 * 1024 : (ctas_per_sm == 3) ? 74 * 1024 : 55 * 1024;
    CK(cudaFuncSetAttribute(k_gather<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    CK(cudaFuncSetAttribute(k_gather<K>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    int occ = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_gather<K>, 256, smem));
    const int blocks = sms * ctas_per_sm;
    CK(cudaMemset(d_cyc, 0, 8));
    k_gather<K><<<blocks, 256, smem>>>(table, entries, 20, spread, noalloc, d_cyc, d_sink);   // warm L2
    CK(cudaMemset(d_cyc, 0, 8));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    CK(cudaEventRecord(e0));
    k_gather<K><<<blocks, 256, smem>>>(table, entries, phases, spread, noalloc, d_cyc, d_sink);
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    unsigned long long cyc = 0;
    CK(cudaMemcpy(&cyc, d_cyc, 8, cudaMemcpyDeviceToHost));
    const double cyc_per_phase = (double)cyc / blocks / phases;                       // as seen by one CTA
    const double sectors = (double)blocks * 256 * K * phases;
    const double gbs = sectors * 32 / (ms * 1e-3) / 1e9;
    const double sm_cycles = (double)cyc / blocks;                                    // kernel duration in SM clocks
    printf("K=%2d ctas/SM=%d(occ %d) spread=%5d noalloc=%d : %7.0f cycles/phase/CTA  %6.2f sectors/clk/SM  %7.0f GB/s  (%.2f ms)\n", K, ctas_per_sm, occ,
           spread, noalloc, cyc_per_phase, sectors / sms / sm_cycles, gbs, ms);
    fflush(stdout);
}

int main() {
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    const int sms = prop.multiProcessorCount;
    const uint32_t entries = 903480;                       // the May 3-D grid: 903 480 entries x 32 B = 29 MB (fp16 octs)
    uint4 *table;
    CK(cudaMalloc(&table, (size_t)entries * 32));
    CK(cudaMemset(table, 1, (size_t)entries * 32));
    unsigned long long *d_cyc; uint32_t *d_sink;
    CK(cudaMalloc(&d_cyc, 8)); CK(cudaMalloc(&d_sink, 4));
    printf("%s, %d SMs; table %u entries x 32 B; one phase = K loads per thread, 256 threads per CTA, CTA barrier\n", prop.name, sms, entries);
    for (int noalloc = 0; noalloc <= 1; ++noalloc)
        for (int spread : {0, 64}) {
            run<8>(table, entries, 1, spread, noalloc, sms, d_cyc, d_sink);
            run<8>(table, entries, 2, spread, noalloc, sms, d_cyc, d_sink);
            run<8>(table, entries, 4, spread, noalloc, sms, d_cyc, d_sink);
        }
    run<1>(table, entries, 2, 0, 1, sms, d_cyc, d_sink);
    run<2>(table, entries, 2, 0, 1, sms, d_cyc, d_sink);
    run<4>(table, entries, 2, 0, 1, sms, d_cyc, d_sink);
    run<16>(table, entries, 2, 0, 1, sms, d_cyc, d_sink);
    return 0;
}
