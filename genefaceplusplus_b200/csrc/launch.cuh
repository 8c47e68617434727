// launch.cuh -- launch helpers: grids are sized in multiples of the SM count (132 on H100) and
// kernels are grid-stride, so a launch is never a ragged fraction of a wave.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace gfpp {

// SM count of the CURRENT device (one process may drive several GPUs: nothing here is cached process-wide).
inline int sm_count() {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
        return n;
    return 148;
}

// blocks for a grid-stride kernel over n items: enough to cover n, capped at 8 resident waves,
// rounded up to a multiple of the SM count when more than one wave is needed.
inline unsigned grid_for(uint64_t n, unsigned threads) {
    const uint64_t need = (n + threads - 1) / threads;
    const uint64_t sms = (uint64_t)sm_count();
    if (need <= sms) return (unsigned)(need ? need : 1);
    uint64_t waves = (need + sms - 1) / sms;
    if (waves > 16) waves = 16;
    return (unsigned)(waves * sms);
}

}  // namespace gfpp
