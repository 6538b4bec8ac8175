// emu_journal.cpp — TEST-ONLY host driver of the drains' kernels under tests/emu/cuda_shim.h: the change scan k_changes
// (limitador_b200/csrc/rl_maint.cuh) and the dictionary drain's mark k_counter_vars_since (rl_cvars_dev.cuh), the SAME
// kernel source the GPU runs, one CUDA thread after the other in a shuffled order.  Not shipped, not a fallback.  The
// call sequence follows rl_counters_drain's delta path in rl_maint.cu: count, and emit only when the count fits.
#include "cuda_shim.h"
// (the shim must come first: it defines __global__ & co. away)
#include <vector>

#include "../../limitador_b200/csrc/rl_cvars_dev.cuh"
#include "../../limitador_b200/csrc/rl_maint.cuh"

extern "C" {

void emu_seed(uint64_t s) { shim_seed = s; }

// rows / shadow: nrows rows of 16 * (1 + cells) bytes; desc: RlCellDesc[groups * 8]; present: [limits].  Returns the
// entries found; they are written (and the shadow brought up to date) only when they fit in cap.
uint64_t emu_changes(const uint8_t* rows, uint8_t* shadow, uint32_t cells, uint64_t nrows, const RlCellDesc* desc,
                     const uint8_t* present, uint64_t cap, uint32_t* out_limit_id, uint64_t* out_key_lo, uint64_t* out_key_hi,
                     uint64_t* out_value, uint64_t* out_expiry) {
    const RlChangeTab T{rows, shadow, 16u * (1 + cells), cells, nrows, desc, present};
    const uint32_t threads = 256, blocks = (uint32_t)((nrows + threads - 1) / threads);
    unsigned long long cnt = 0;
    RlChangeOut O{nullptr, nullptr, nullptr, nullptr, nullptr, &cnt};
    shim_launch(blocks, threads, [&] { k_changes(T, O, 0); });
    if (cnt > cap) return cnt;
    const unsigned long long found = cnt;
    cnt = 0;
    O = RlChangeOut{out_limit_id, out_key_lo, out_key_hi, out_value, out_expiry, &cnt};
    shim_launch(blocks, threads, [&] { k_changes(T, O, 1); });
    return found;
}

// mark[p] for the nslots slots (a power of two), as rl_cv_dev_drain launches it
void emu_cv_since(CvSlot* slots, uint64_t nslots, uint64_t since, uint8_t* mark) {
    const CvDict d{slots, nslots - 1, nullptr, 0, nullptr};
    shim_launch((uint32_t)((nslots + 255) / 256), 256, [&] { k_counter_vars_since(d, since, mark); });
}

}  // extern "C"
