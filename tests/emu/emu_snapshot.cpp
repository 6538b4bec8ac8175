// emu_snapshot.cpp — TEST-ONLY host driver of the counter-import kernels (limitador_b200/csrc/rl_maint.cuh:
// k_import_resolve, k_import_claim, k_import_write) under tests/emu/cuda_shim.h: the SAME kernel source the GPU runs,
// one CUDA thread after the other in a shuffled order.  Not shipped, not a fallback.  The launch geometry and the pass
// sequence follow rl_counters_import (rl_maint.cu).
// Built twice: plain (cuda_shim.h) and with -DEMU_SIMT (cuda_simt.h: the threads of a block as fibers, so that the
// warp-aggregated probe of k_import_claim runs).
#ifdef EMU_SIMT
#include "cuda_simt.h"
#define shim_launch simt_launch
static uint64_t shim_seed = 0;
#else
#include "cuda_shim.h"
#endif
// (the shim must come first: it defines __global__ & co. away)
#include <vector>

#include "../../limitador_b200/csrc/rl_maint.cuh"

extern "C" {

void emu_seed(uint64_t s) { shim_seed = s; }

// rows: the table (capacity = 2^(log2P + log2R) rows of 16 * (1 + cells) bytes), changed in place; limits:
// RlLimitDev[limits_cap].  Returns the error word ((index << 8) | reason, ~0 = imported); unq_out[limits_cap] = the
// unqualified limits the call makes present.
unsigned long long emu_import(uint8_t* rows, uint32_t cells, uint32_t log2P, uint32_t log2R, const RlLimitDev* limits,
                              uint32_t limits_cap, uint64_t n, const uint32_t* limit_id, const uint64_t* key_lo,
                              const uint64_t* key_hi, const uint64_t* value, const uint64_t* expiry_us,
                              uint8_t* unq_out) {
    const RlImportTab T{rows, 16u * (1 + cells), log2P, log2R, limits, limits_cap};
    const RlImportIn I{limit_id, key_lo, key_hi, value, expiry_us, n};
    const uint64_t capacity = 1ull << (log2P + log2R);
    unsigned long long err = ~0ull;
    std::vector<uint8_t> unq(limits_cap, 0);
    const uint32_t threads = 256, blocks = (uint32_t)((n + threads - 1) / threads);
    if (n == 0) return err;
    shim_launch(blocks, threads, [&] { k_import_resolve(T, I, &err, unq.data()); });
    if (err != ~0ull) return err;
    std::vector<unsigned long long> row_of(n, 0);
    std::vector<unsigned> mask(capacity, 0);
    shim_launch(blocks, threads, [&] { k_import_claim(T, I, row_of.data(), mask.data(), &err); });
    if (err != ~0ull) {
        shim_launch(blocks, threads, [&] { k_import_release(T, n, row_of.data()); });
        return err;
    }
    shim_launch(blocks, threads, [&] { k_import_write(T, I, row_of.data()); });
    for (uint32_t l = 0; l < limits_cap; l++) unq_out[l] = unq[l];
    return err;
}

}  // extern "C"
