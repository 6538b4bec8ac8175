// simt_selftest.cpp — the fiber emulator (cuda_simt.h) checked on its own: results of the warp intrinsics and the block
// barrier against closed forms, and — run with an argument — the three mistakes it must refuse (they are hangs or undefined
// behaviour on a GPU): a *_sync mask naming an exited lane, lanes disagreeing on the mask, a barrier not every thread reaches.
// Also the interleaving mode: a read-modify-write made of a plain load and store with a switch point between them must lose
// updates under it, and the same update as an atomic must not — the mode can show a race at all.  And what the decision
// kernels need: __shfl_up_sync scans, the reducing barriers, atomicOr, min / max on mixed types, uint4, static
// __shared__ arrays, per-block dynamic shared memory that starts poisoned, and resident blocks: block 0 waits in a
// __nanosleep loop for a flag block 1 sets, which finishes with two resident blocks and is reported as a hang with one.
#include "cuda_simt.h"

#include <cstdio>
#include <cstring>
#include <vector>

static unsigned g_smem[256];

__global__ void k_ok(unsigned* out_match, unsigned* out_sum, unsigned* out_ballot, unsigned* out_block_sum, unsigned* out_shfl) {
    const unsigned t = threadIdx.x, lane = t & 31u;
    const unsigned key = t % 5;  // five groups per warp
    const unsigned grp = __match_any_sync(0xFFFFFFFFu, key);
    out_match[blockIdx.x * blockDim.x + t] = grp;
    out_sum[blockIdx.x * blockDim.x + t] = __reduce_add_sync(grp, t);  // every group reduces over its own mask
    out_ballot[blockIdx.x * blockDim.x + t] = __ballot_sync(0xFFFFFFFFu, lane % 3 == 0);
    out_shfl[blockIdx.x * blockDim.x + t] = __shfl_sync(0xFFFFFFFFu, t * 10, (lane + 1) & 31);
    // block-wide tree reduction through a shared array: every step separated by the barrier
    g_smem[t] = t + 1;
    __syncthreads();
    for (unsigned s = blockDim.x / 2; s > 0; s >>= 1) {
        if (t < s) g_smem[t] += g_smem[t + s];
        __syncthreads();
    }
    if (t == 0) out_block_sum[blockIdx.x] = g_smem[0];
    __syncthreads();  // nobody overwrites g_smem for the next block's use before thread 0 has read it (blocks run in turn)
}

__global__ void k_racy_inc(unsigned long long* counter) {
    const unsigned long long v = *counter;  // plain load ...
    simt::interleave_point();
    *counter = v + 1;                       // ... and plain store: another fiber's update in between is lost
}
__global__ void k_atomic_inc(unsigned long long* counter) { atomicAdd(counter, 1ull); }

// the two counters after one 256-thread block of each kernel under the interleaving mode
static void race(uint64_t seed, double p, unsigned long long* racy, unsigned long long* atomic) {
    *racy = *atomic = 0;
    simt_interleave(true, seed, p);
    simt_launch(1, 256, [&] { k_racy_inc(racy); });
    simt_launch(1, 256, [&] { k_atomic_inc(atomic); });
    simt_interleave(false);
}

__global__ void k_exited_lane() {
    if ((threadIdx.x & 31u) == 7) return;  // lane 7 leaves ...
    __ballot_sync(0xFFFFFFFFu, 1);         // ... and the others name it
}
__global__ void k_mask_mismatch() {
    const unsigned lane = threadIdx.x & 31u;
    __reduce_add_sync(lane < 16 ? 0x0000FFFFu : 0xFFFFFFFFu, 1u);  // the upper half names lanes that brought another mask
}
__global__ void k_missed_barrier() {
    if (threadIdx.x != 3) __syncthreads();
    if (threadIdx.x == 3) __syncwarp(1u << 3);
    __syncthreads();
    if (threadIdx.x == 5) return;
    __syncthreads();
    // thread 3 skipped the first barrier: the counts no longer line up and somebody waits for ever
    if (threadIdx.x & 1) __syncthreads();
}

// inclusive scan of the lane ids with __shfl_up_sync, the reducing barriers, atomicOr, static __shared__, uint4, min/max
__global__ void k_scan_reduce(unsigned* out_scan, int* out_or, int* out_and, unsigned* out_bits, uint4* out_q) {
    __shared__ unsigned s_bits;
    const unsigned t = threadIdx.x, lane = t & 31u;
    if (t == 0) s_bits = 0;
    __syncthreads();
    unsigned x = lane + 1;
    for (unsigned o = 1; o < 32; o <<= 1) {
        const unsigned y = __shfl_up_sync(0xFFFFFFFFu, x, o);
        if (lane >= o) x += y;
    }
    out_scan[blockIdx.x * blockDim.x + t] = x;
    out_or[blockIdx.x * 2 + 0] = __syncthreads_or(t == 77);    // one thread true
    out_or[blockIdx.x * 2 + 1] = __syncthreads_or(0);          // none
    out_and[blockIdx.x * 2 + 0] = __syncthreads_and(t != 77);  // one thread false
    out_and[blockIdx.x * 2 + 1] = __syncthreads_and(1);        // all
    atomicOr(&s_bits, 1u << (t & 31u));
    __syncthreads();
    if (t == 0) {
        *out_bits = s_bits;
        const uint64_t big = 1ull << 40;
        *out_q = make_uint4(min(3u, big), (unsigned)(max(2u, big) >> 32), min(blockDim.x, 7u), max(1, -1));
    }
}

// dynamic shared memory: every block must find it poisoned (not the previous block's values), then owns it
__global__ void k_dyn_smem(unsigned* out_fresh) {
    unsigned* s = reinterpret_cast<unsigned*>(simt_dyn_smem());
    const unsigned t = threadIdx.x;
    const bool poisoned = s[t] == 0xA5A5A5A5u;
    __syncthreads();
    s[t] = blockIdx.x + 1;  // what a block that saw its predecessor's memory would read
    __syncthreads();
    if (s[(t + 1) % blockDim.x] != blockIdx.x + 1) out_fresh[blockIdx.x] = 2;
    if (!__syncthreads_and(poisoned) && t == 0) out_fresh[blockIdx.x] = 3;
}

// block 0 waits for a flag that block 1 sets: finishes only if both are resident at once
__global__ void k_flag_wait(volatile unsigned* flag, unsigned* seen) {
    if (blockIdx.x == 1) {
        __syncthreads();
        if (threadIdx.x == 0) {
            __threadfence();
            __threadfence_system();  // a switch point like __threadfence (the peer exchange's kernels fence at system scope)
            atomicExch(const_cast<unsigned*>(flag), 1u);
        }
        return;
    }
    for (;;) {
        if (__syncthreads_or(*flag != 0)) break;
        __nanosleep(100);
    }
    if (threadIdx.x == 0) *seen = 1;
}

int main(int argc, char** argv) {
    if (argc > 1) {
        if (!strcmp(argv[1], "spin")) {  // the flag wait with one resident block: the detector must report it
            unsigned flag = 0, seen = 0;
            simt_launch_ex(2, 64, 0, 1, [&] { k_flag_wait(&flag, &seen); });
        }
        if (!strcmp(argv[1], "exited")) simt_launch(1, 64, [] { k_exited_lane(); });
        if (!strcmp(argv[1], "mask")) simt_launch(1, 32, [] { k_mask_mismatch(); });
        if (!strcmp(argv[1], "barrier")) simt_launch(1, 32, [] { k_missed_barrier(); });
        printf("not refused\n");
        return 0;
    }
    const unsigned grid = 3, block = 128, n = grid * block;
    std::vector<unsigned> m(n), s(n), b(n), bs(grid), sh(n);
    simt_launch(grid, block, [&] { k_ok(m.data(), s.data(), b.data(), bs.data(), sh.data()); });
    for (unsigned i = 0; i < n; i++) {
        const unsigned t = i % block, lane = t & 31u, w0 = t - lane;
        unsigned grp = 0, sum = 0, ballot = 0;
        for (unsigned j = 0; j < 32; j++) {
            if ((w0 + j) % 5 == t % 5) {
                grp |= 1u << j;
                sum += w0 + j;
            }
            if (j % 3 == 0) ballot |= 1u << j;
        }
        if (m[i] != grp || s[i] != sum || b[i] != ballot || sh[i] != (w0 + ((lane + 1) & 31)) * 10) return 2;
    }
    for (unsigned g = 0; g < grid; g++)
        if (bs[g] != block * (block + 1) / 2) return 3;
    // interleaving mode off (the default): every thread runs to its end, the racy update loses nothing
    unsigned long long racy = 0, atomic = 0;
    simt_launch(1, 256, [&] { k_racy_inc(&racy); });
    if (racy != 256) return 4;
    // on: the racy update loses some increments, whether every switch point switches or half of them do; the atomic none
    race(1, 1.0, &racy, &atomic);
    if (racy >= 256 || atomic != 256) return 5;
    const unsigned long long lost_p1 = 256 - racy;
    race(2, 0.5, &racy, &atomic);
    if (racy >= 256 || atomic != 256) return 6;
    // shfl_up scan, reducing barriers, atomicOr, static __shared__, uint4, mixed min / max
    {
        const unsigned g2 = 2, b2 = 128;
        std::vector<unsigned> scan(g2 * b2);
        int ors[4], ands[4];
        unsigned bits = 0;
        uint4 q{};
        simt_launch(g2, b2, [&] { k_scan_reduce(scan.data(), ors, ands, &bits, &q); });
        for (unsigned i = 0; i < g2 * b2; i++) {
            const unsigned lane = i % 32;
            if (scan[i] != (lane + 1) * (lane + 2) / 2) return 7;
        }
        for (unsigned g = 0; g < g2; g++)
            if (ors[2 * g] != 1 || ors[2 * g + 1] != 0 || ands[2 * g] != 0 || ands[2 * g + 1] != 1) return 8;
        if (bits != 0xFFFFFFFFu || q.x != 3 || q.y != 256 || q.z != 7 || q.w != 1) return 9;
    }
    // dynamic shared memory: poisoned at every block start, one copy per resident block, with one or four resident
    for (unsigned R : {1u, 4u}) {
        std::vector<unsigned> fresh(9, 0);
        simt_launch_ex(9, 64, 64 * sizeof(unsigned), R, [&] { k_dyn_smem(fresh.data()); });
        for (unsigned v : fresh)
            if (v) return 10;
        simt_interleave(true, 7, 1.0);
        simt_launch_ex(9, 64, 64 * sizeof(unsigned), R, [&] { k_dyn_smem(fresh.data()); });
        simt_interleave(false);
        for (unsigned v : fresh)
            if (v) return 11;
    }
    // resident blocks: the flag wait finishes with two of them, in either mode
    {
        unsigned flag = 0, seen = 0;
        simt_launch_ex(2, 64, 0, 2, [&] { k_flag_wait(&flag, &seen); });
        if (!seen) return 12;
        flag = seen = 0;
        simt_interleave(true, 3, 0.5);
        simt_launch_ex(2, 64, 0, 2, [&] { k_flag_wait(&flag, &seen); });
        simt_interleave(false);
        if (!seen) return 13;
    }
    printf("ok simt (racy update lost %llu and %llu of 256 increments)\n", lost_p1, 256 - racy);
    return 0;
}
