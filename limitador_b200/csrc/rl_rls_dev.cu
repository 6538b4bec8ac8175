// rl_rls_dev.cu — host side of the RLS device plan (rl_rls_dev.h; kernels in rl_rls_dev.cuh).  A translation unit of its
// own: it sees an engine only through rl_internal.h and the public C-ABI, and a matcher only through its image.
//
// One plan: wire bytes and offsets -> pinned staging -> device (engine's stream); k_rls_plan; CUB exclusive sum; ONE
// device->host read of the totals (the store request and counter counts); k_rls_scatter; the per-request array back
// into pinned memory.  The store call then reads the CSR where it lies (RL_MEM_DEVICE).  The HTTP plan (rl_http_dev.cuh)
// takes the same path through the same state: staging, image, scratch and the one read are shared, the kernels and the
// per-request array are its own, and its read also brings the table of its store calls.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include <cub/device/device_scan.cuh>
#include <cuda/std/functional>

#include "rl_cuda_host.h"
#include "rl_cvars_dev.cuh"
#include "rl_http_dev.cuh"
#include "rl_internal.h"
#include "rl_rls_dev.cuh"

struct rl_rls_dev {
    int device = 0;
    cudaStream_t stream = nullptr;
    std::string err;
    // the matcher image: host copy (its header places the sections) and device copy
    uint64_t gen = 0;
    std::vector<uint32_t> image;
    DevBuf<uint32_t> d_image;
    // the batch
    uint64_t n = 0, n_store = 0, n_ctr = 0;
    PinnedBuf<uint8_t> h_buf;
    PinnedBuf<uint64_t> h_off;
    PinnedBuf<RlsDevReq> h_req;
    PinnedBuf<unsigned long long> h_total;
    DevBuf<uint8_t> d_buf, d_cub;
    DevBuf<uint64_t> d_off;
    DevBuf<rl_rls_entry> d_ent;
    DevBuf<rl_counter> d_scratch, d_ctrs;
    DevBuf<RlsDevReq> d_req;
    DevBuf<unsigned long long> d_count, d_start;
    DevBuf<uint32_t> d_ctr_off;
    DevBuf<uint64_t> d_delta, d_now;
    // store call outputs
    DevBuf<uint8_t> d_lim;
    DevBuf<uint32_t> d_first;
    DevBuf<uint64_t> d_rem, d_ttl;
    // the HTTP plan's own arrays
    DevBuf<uint8_t> d_txt, d_bits, d_load;
    DevBuf<HttpDevReq> d_hreq;
    PinnedBuf<HttpDevReq> h_hreq;
    DevBuf<HttpScan> d_hcount, d_hstart;
    DevBuf<uint32_t> d_runs, d_ctr_run;
    PinnedBuf<uint32_t> h_runs;
    uint32_t n_runs = 0;
    // the counter variable dictionary (rl_cvars_dev.cuh): off while cv_slots == 0
    uint64_t cv_slots = 0, cv_arena_bytes = 0;
    DevBuf<CvSlot> d_cv_slots;
    DevBuf<uint8_t> d_cv_arena;
    DevBuf<unsigned long long> d_cv_ctl;
    // drains: the arena cursor the last drain read; the next drain is full after keeping is set, a GC or an import
    uint64_t cv_since = 0;
    bool cv_full_next = true;
    // lookup and GC scratch
    DevBuf<uint32_t> d_cv_lid;
    DevBuf<uint64_t> d_cv_lo, d_cv_hi, d_cv_val, d_cv_exp, d_cv_src;
    DevBuf<unsigned long long> d_cv_len, d_cv_pos;
    DevBuf<unsigned long long> d_cv_idx;  // export: each entry's index
    DevBuf<uint8_t> d_cv_mark, d_cv_out;
    std::vector<unsigned long long> h_cv_pos;
    std::vector<uint64_t> h_cv_src;
    std::vector<uint8_t> h_cv_out, h_cv_unnamed;
};

namespace {

template <class... A>
int fail(rl_rls_dev* S, int status, const char* fmt, A... a) {
    S->err = rl_format(fmt, a...);
    return status;
}

uint32_t blocks_for(uint64_t n, uint32_t threads) { return (uint32_t)((n + threads - 1) / threads); }

// upload the matcher's image when its generation moved since the last batch
int refresh_image(rl_rls_dev* S, rl_matcher* m) {
    const uint64_t g = rl_matcher_generation(m);
    if (g == S->gen && !S->image.empty()) return RL_OK;
    if (S->image.size() < 1024) S->image.resize(1024);
    uint64_t need = 0, got = 0;
    while (rl_matcher_image(m, S->image.data(), S->image.size(), &need, &got) != RL_OK) {
        if (need <= S->image.size()) return fail(S, RL_FATAL, "the matcher image could not be taken");
        S->image.resize(need);
    }
    S->image.resize(need);
    RL_CUDA(S, S->d_image.grow(need));
    RL_CUDA(S, cudaMemcpyAsync(S->d_image.p, S->image.data(), need * sizeof(uint32_t), cudaMemcpyHostToDevice, S->stream));
    S->gen = got;
    return RL_OK;
}


// What both plans start with: the engine's device and stream, the matcher image, the batch's bytes and offsets through
// pinned staging onto the device, and the entry and counter scratch.  per_req = counters one request may carry.
int stage_batch(rl_rls_dev* S, rl_engine* e, rl_matcher* m, uint64_t n, const uint8_t* buf, const uint64_t* off,
                uint32_t& per_req) {
    S->n = S->n_store = S->n_ctr = 0;
    S->n_runs = 0;
    RlTableView v;
    int r = rl_internal_view(e, &v);  // the engine's device and stream (every earlier pipelined call is fenced)
    if (r) return fail(S, r, "%s", rl_last_error(e));
    S->device = v.device;
    S->stream = v.stream;
    if ((r = refresh_image(S, m))) return r;
    const uint32_t engine_max = rl_engine_max_counters_per_request(e);
    per_req = std::min(S->image[RL_IMG_H_COUNTER_CAP], engine_max);
    if (n && (n + 1) * (uint64_t)per_req >= (1ull << 32))
        return fail(S, RL_FATAL, "a batch of %llu requests of up to %u counters each may exceed 2^32 counters",
                        (unsigned long long)n, per_req);
    const uint64_t bytes = n ? off[n] : 0;
    // wire bytes and offsets through pinned staging onto the device
    RL_CUDA(S, S->h_buf.grow(bytes + 1));
    RL_CUDA(S, S->h_off.grow(n + 1));
    RL_CUDA(S, S->h_total.grow(1));
    if (bytes) memcpy(S->h_buf.p, buf, bytes);
    memcpy(S->h_off.p, off, (n + 1) * sizeof(uint64_t));
    RL_CUDA(S, S->d_buf.grow(bytes + 1));
    RL_CUDA(S, S->d_off.grow(n + 1));
    RL_CUDA(S, S->d_ent.grow(bytes / 2 + 1));
    RL_CUDA(S, S->d_scratch.grow(n * (uint64_t)per_req + 1));
    if (bytes) RL_CUDA(S, cudaMemcpyAsync(S->d_buf.p, S->h_buf.p, bytes, cudaMemcpyHostToDevice, S->stream));
    RL_CUDA(S, cudaMemcpyAsync(S->d_off.p, S->h_off.p, (n + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, S->stream));
    return RL_OK;
}

// the one read before the store call: `bytes` from the device to pinned host memory, then the stream is waited for
int read_totals(rl_rls_dev* S, void* dst, const void* src, size_t bytes) {
    RL_CUDA(S, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, S->stream));
    RL_CUDA(S, cudaStreamSynchronize(S->stream));
    return RL_OK;
}

// the store call's outputs from the device arrays to the caller's (with load_counters also the CSR the headers read)
int copy_outputs(rl_rls_dev* S, bool verdicts, bool load_counters, uint8_t* limited, uint32_t* first_limited,
                 uint64_t* remaining, uint64_t* ttl_us, uint32_t* ctr_off, rl_counter* ctrs) {
    const uint64_t m = S->n_store, nc = S->n_ctr;
    if (verdicts) {
        if (cudaMemcpyAsync(limited, S->d_lim.p, m, cudaMemcpyDeviceToHost, S->stream) != cudaSuccess ||
            cudaMemcpyAsync(first_limited, S->d_first.p, m * sizeof(uint32_t), cudaMemcpyDeviceToHost, S->stream) != cudaSuccess)
            return fail(S, RL_FATAL, "copying the verdicts back failed");
    }
    if (load_counters) {
        if (cudaMemcpyAsync(remaining, S->d_rem.p, nc * sizeof(uint64_t), cudaMemcpyDeviceToHost, S->stream) != cudaSuccess ||
            cudaMemcpyAsync(ttl_us, S->d_ttl.p, nc * sizeof(uint64_t), cudaMemcpyDeviceToHost, S->stream) != cudaSuccess ||
            cudaMemcpyAsync(ctr_off, S->d_ctr_off.p, (m + 1) * sizeof(uint32_t), cudaMemcpyDeviceToHost, S->stream) != cudaSuccess ||
            cudaMemcpyAsync(ctrs, S->d_ctrs.p, nc * sizeof(rl_counter), cudaMemcpyDeviceToHost, S->stream) != cudaSuccess)
            return fail(S, RL_FATAL, "copying the counters back failed");
    }
    return RL_OK;
}

// the store call's output buffers; with load_counters remaining / ttl start at 0 (slots of a refused call stay 0, as
// with host buffers)
int reserve_outputs(rl_rls_dev* S, bool load_counters) {
    const uint64_t m = S->n_store, nc = S->n_ctr;
    RL_CUDA(S, S->d_lim.grow(m));
    RL_CUDA(S, S->d_first.grow(m));
    if (load_counters) {
        RL_CUDA(S, S->d_rem.grow(nc + 1));
        RL_CUDA(S, S->d_ttl.grow(nc + 1));
        RL_CUDA(S, cudaMemsetAsync(S->d_rem.p, 0, (nc + 1) * sizeof(uint64_t), S->stream));
        RL_CUDA(S, cudaMemsetAsync(S->d_ttl.p, 0, (nc + 1) * sizeof(uint64_t), S->stream));
    }
    return RL_OK;
}

// The engine call a store request makes: RLS method or HTTP endpoint -> operation
enum StoreOp { CHECK_AND_UPDATE, IS_WITHIN, UPDATE };
StoreOp store_op(bool http, int method) {
    if (http) return method == RL_HTTP_CHECK_AND_REPORT ? CHECK_AND_UPDATE : method == RL_HTTP_CHECK ? IS_WITHIN : UPDATE;
    return method == RL_RLS_SHOULD_RATE_LIMIT ? CHECK_AND_UPDATE : method == RL_RLS_CHECK_RATE_LIMIT ? IS_WITHIN : UPDATE;
}

// One store call on the device arrays: the m store requests from j0, whose CSR offsets `off` count from counter c0.
// Returns its status, with the device-memory call's deferred errors.
int store_call(rl_rls_dev* S, rl_engine* e, StoreOp op, uint64_t j0, uint64_t m, const uint32_t* off, uint64_t c0, bool load) {
    const rl_counter* c = S->d_ctrs.p + c0;
    const uint64_t *d = S->d_delta.p + j0, *now = S->d_now.p + j0;
    int st;
    if (op == CHECK_AND_UPDATE)
        st = rl_check_and_update_batch(e, m, off, c, d, now, load, RL_MEM_DEVICE, S->d_lim.p + j0, S->d_first.p + j0,
                                       load ? S->d_rem.p + c0 : nullptr, load ? S->d_ttl.p + c0 : nullptr);
    else if (op == IS_WITHIN)
        st = rl_is_within_limits_batch(e, m, off, c, d, now, RL_MEM_DEVICE, S->d_lim.p + j0, S->d_first.p + j0);
    else
        st = rl_update_batch(e, m, off, c, d, now, RL_MEM_DEVICE);
    return st == RL_OK ? rl_sync(e) : st;
}

// The store call's CSR on the device, once the plan read its size: ctr_off [n_store + 1], ctrs [n_ctr], delta and now
// [n_store]
int grow_csr(rl_rls_dev* S, uint64_t n_store, uint64_t n_ctr) {
    RL_CUDA(S, S->d_ctr_off.grow(n_store + 1));
    RL_CUDA(S, S->d_ctrs.grow(n_ctr + 1));
    RL_CUDA(S, S->d_delta.grow(n_store + 1));
    RL_CUDA(S, S->d_now.grow(n_store + 1));
    return RL_OK;
}

// What both plans end with: the per-request array back into pinned memory (there once the stream is waited for), the
// batch's sizes and the out-parameters.
template <class Req>
int close_plan(rl_rls_dev* S, uint64_t n, uint64_t n_store, uint64_t n_ctr, PinnedBuf<Req>& h_req, const DevBuf<Req>& d_req,
               uint64_t* out_n_store, uint64_t* out_n_ctr, const Req** out_req) {
    if (n) RL_CUDA(S, cudaMemcpyAsync(h_req.p, d_req.p, n * sizeof(Req), cudaMemcpyDeviceToHost, S->stream));
    S->n = n;
    S->n_store = n_store;
    S->n_ctr = n_ctr;
    *out_n_store = n_store;
    *out_n_ctr = n_ctr;
    *out_req = h_req.p;
    return RL_OK;
}

CvDict cv_dict(rl_rls_dev* S) {
    return CvDict{S->d_cv_slots.p, S->cv_slots - 1, S->d_cv_arena.p, S->cv_arena_bytes, S->d_cv_ctl.p};
}

// k_counter_vars_record after a plan's scatter, when keeping is on: the plan's scratch is still the batch's.  Then the
// plan's `launched` kernels and this one are counted.
template <class Dec>
int record_vars(rl_rls_dev* S, rl_engine* e, uint32_t launched, uint64_t n, uint32_t per_req, const unsigned long long* rls_count,
                const HttpScan* http_count) {
    if (S->cv_slots && n) {
        CvRecordArgs a;
        a.buf = S->d_buf.p;
        a.off = S->d_off.p;
        a.n = n;
        a.img = rl_img_view(S->image.data(), S->d_image.p);
        a.per_req = per_req;
        a.ent = S->d_ent.p;
        a.scratch = S->d_scratch.p;
        a.rls_count = rls_count;
        a.http_count = http_count;
        a.txt = S->d_txt.p;
        a.bits = S->d_bits.p;
        a.dict = cv_dict(S);
        const uint32_t threads = 128;
        k_counter_vars_record<Dec><<<blocks_for(n, threads), threads, 0, S->stream>>>(a);
        RL_CUDA(S, cudaGetLastError());
        launched++;
    }
    rl_internal_launched(e, launched);
    return RL_OK;
}

// The first half of the GC and of the export: the engine's counters rl_counters_export(ns_ids, now_us) lists, on the
// device, and the dictionary slots they reference marked in d_cv_mark [slots + 1] (mark[slots] = 0: the export scans
// it).  d_cv_len and d_cv_pos get room for kept_positions.  launched = the kernels run (0 or 1).
int mark_live(rl_rls_dev* S, rl_engine* e, const uint32_t* ns_ids, uint32_t n_ns, uint64_t now_us, uint32_t& launched) {
    launched = 0;
    uint64_t n = 0;
    int r;
    if ((r = rl_counters_export(e, ns_ids, n_ns, now_us, 0, RL_MEM_DEVICE, nullptr, nullptr, nullptr, nullptr, nullptr, &n)))
        return fail(S, r, "%s", rl_last_error(e));
    RL_CUDA(S, S->d_cv_lid.grow(n + 1));
    RL_CUDA(S, S->d_cv_lo.grow(n + 1));
    RL_CUDA(S, S->d_cv_hi.grow(n + 1));
    RL_CUDA(S, S->d_cv_val.grow(n + 1));
    RL_CUDA(S, S->d_cv_exp.grow(n + 1));
    uint64_t got = 0;
    if ((r = rl_counters_export(e, ns_ids, n_ns, now_us, n, RL_MEM_DEVICE, S->d_cv_lid.p, S->d_cv_lo.p, S->d_cv_hi.p, S->d_cv_val.p,
                                S->d_cv_exp.p, &got)))
        return fail(S, r, "%s", rl_last_error(e));
    n = std::min(n, got);
    const uint64_t slots = S->cv_slots;
    RL_CUDA(S, S->d_cv_mark.grow(slots + 1));
    RL_CUDA(S, S->d_cv_len.grow(slots + 1));
    RL_CUDA(S, S->d_cv_pos.grow(slots + 1));
    RL_CUDA(S, cudaMemsetAsync(S->d_cv_mark.p, 0, slots + 1, S->stream));
    if (n) {
        const uint32_t threads = 256;
        CvMarkArgs a{S->d_cv_lid.p, S->d_cv_lo.p, S->d_cv_hi.p, n, rl_img_view(S->image.data(), S->d_image.p), cv_dict(S), S->d_cv_mark.p};
        k_counter_vars_mark<<<blocks_for(n, threads), threads, 0, S->stream>>>(a);
        RL_CUDA(S, cudaGetLastError());
        launched = 1;
    }
    return RL_OK;
}

// d_cv_pos = where each marked slot's blob goes in a compacted arena (d_cv_pos[slots] = the kept bytes): one kernel
int kept_positions(rl_rls_dev* S) {
    const uint64_t slots = S->cv_slots;
    const uint32_t threads = 256;
    k_counter_vars_kept<<<blocks_for(slots + 1, threads), threads, 0, S->stream>>>(cv_dict(S), S->d_cv_mark.p, S->d_cv_len.p);
    RL_CUDA(S, cudaGetLastError());
    size_t tmp = 0;
    RL_CUDA(S, cub::DeviceScan::ExclusiveSum(nullptr, tmp, S->d_cv_len.p, S->d_cv_pos.p, (int64_t)(slots + 1), S->stream));
    RL_CUDA(S, S->d_cub.grow(tmp + 1));
    RL_CUDA(S, cub::DeviceScan::ExclusiveSum(S->d_cub.p, tmp, S->d_cv_len.p, S->d_cv_pos.p, (int64_t)(slots + 1), S->stream));
    return RL_OK;
}

// The marked entries copied into a fresh table and arena of the configured sizes (the count of dropped keys carries
// over): one kernel.  The caller swaps them in.
int rebuild_fresh(rl_rls_dev* S, DevBuf<CvSlot>& slots2, DevBuf<uint8_t>& arena2, DevBuf<unsigned long long>& ctl2) {
    const uint64_t slots = S->cv_slots;
    RL_CUDA(S, slots2.exact(slots));
    RL_CUDA(S, arena2.exact(S->cv_arena_bytes));
    RL_CUDA(S, ctl2.exact(RL_CV_CTL_WORDS));
    RL_CUDA(S, cudaMemsetAsync(slots2.p, 0, slots * sizeof(CvSlot), S->stream));
    RL_CUDA(S, cudaMemsetAsync(ctl2.p, 0, RL_CV_CTL_WORDS * sizeof(unsigned long long), S->stream));
    RL_CUDA(S, cudaMemcpyAsync(ctl2.p + RL_CV_DROPPED, S->d_cv_ctl.p + RL_CV_DROPPED, sizeof(unsigned long long),
                                cudaMemcpyDeviceToDevice, S->stream));
    CvRebuildArgs b{cv_dict(S), S->d_cv_mark.p, S->d_cv_pos.p, CvDict{slots2.p, slots - 1, arena2.p, S->cv_arena_bytes, ctl2.p}};
    const uint32_t threads = 256;
    k_counter_vars_rebuild<<<blocks_for(slots + 1, threads), threads, 0, S->stream>>>(b);
    RL_CUDA(S, cudaGetLastError());
    return RL_OK;
}

// The second half of the export and of the drains: the slots marked in d_cv_mark [slots + 1] laid out for the host.
// *out_count / *out_bytes = what the marks select; written only when cap and bytes_cap hold it all.
int export_marked(rl_rls_dev* S, rl_engine* e, uint64_t cap, uint64_t bytes_cap, uint32_t* out_varset, uint64_t* out_key_lo,
                  uint64_t* out_key_hi, uint64_t* out_blob_off, uint8_t* out_blobs, uint64_t* out_count, uint64_t* out_bytes) {
    int r;
    if ((r = kept_positions(S))) return r;
    // each entry's index: a scan over the marks
    const uint64_t slots = S->cv_slots;
    RL_CUDA(S, S->d_cv_idx.grow(slots + 1));
    size_t tmp = 0;
    RL_CUDA(S, cub::DeviceScan::ExclusiveScan(nullptr, tmp, S->d_cv_mark.p, S->d_cv_idx.p, cuda::std::plus<>(), 0ull, (int64_t)(slots + 1),
                                               S->stream));
    RL_CUDA(S, S->d_cub.grow(tmp + 1));
    RL_CUDA(S, cub::DeviceScan::ExclusiveScan(S->d_cub.p, tmp, S->d_cv_mark.p, S->d_cv_idx.p, cuda::std::plus<>(), 0ull,
                                               (int64_t)(slots + 1), S->stream));
    unsigned long long tot[2] = {0, 0};
    RL_CUDA(S, cudaMemcpyAsync(&tot[0], S->d_cv_idx.p + slots, sizeof tot[0], cudaMemcpyDeviceToHost, S->stream));
    RL_CUDA(S, cudaMemcpyAsync(&tot[1], S->d_cv_pos.p + slots, sizeof tot[1], cudaMemcpyDeviceToHost, S->stream));
    RL_CUDA(S, cudaStreamSynchronize(S->stream));
    rl_internal_launched(e, 1);
    const uint64_t count = tot[0], bytes = tot[1];
    *out_count = count;
    *out_bytes = bytes;
    if (cap == 0 || cap < count || bytes_cap < bytes) return RL_OK;
    if (!out_varset || !out_key_lo || !out_key_hi || !out_blob_off || (bytes && !out_blobs))
        return fail(S, RL_FATAL, "exporting counter variables: cap > 0 needs every output array");
    // one packed array on the device, one copy to the host: varset (padded to 8 bytes), key_lo, key_hi, blob_off, blobs
    const uint64_t o_lo = (4 * count + 7) / 8 * 8, o_hi = o_lo + 8 * count, o_off = o_hi + 8 * count, o_blob = o_off + 8 * (count + 1);
    RL_CUDA(S, S->d_cv_out.grow(o_blob + bytes));
    uint8_t* P = S->d_cv_out.p;
    CvExportArgs a{cv_dict(S), S->d_cv_mark.p, S->d_cv_pos.p, S->d_cv_idx.p, reinterpret_cast<uint32_t*>(P),
                   reinterpret_cast<uint64_t*>(P + o_lo), reinterpret_cast<uint64_t*>(P + o_hi),
                   reinterpret_cast<uint64_t*>(P + o_off), P + o_blob};
    const uint32_t threads = 256;
    k_counter_vars_export<<<blocks_for(slots + 1, threads), threads, 0, S->stream>>>(a);
    RL_CUDA(S, cudaGetLastError());
    rl_internal_launched(e, 1);
    S->h_cv_out.resize(o_blob + bytes);
    RL_CUDA(S, cudaMemcpyAsync(S->h_cv_out.data(), P, o_blob + bytes, cudaMemcpyDeviceToHost, S->stream));
    RL_CUDA(S, cudaStreamSynchronize(S->stream));
    const uint8_t* h = S->h_cv_out.data();
    memcpy(out_varset, h, 4 * count);
    memcpy(out_key_lo, h + o_lo, 8 * count);
    memcpy(out_key_hi, h + o_hi, 8 * count);
    memcpy(out_blob_off, h + o_off, 8 * (count + 1));
    if (bytes) memcpy(out_blobs, h + o_blob, bytes);
    return RL_OK;
}


const char* cv_reason(uint64_t why) {
    switch (why) {
        case RL_CV_BAD_VARSET: return "not the variable set of a qualified limit";
        case RL_CV_BAD_LENGTH: return "a length runs past the blob";
        case RL_CV_BAD_TRAILING: return "bytes after the last value";
        case RL_CV_BAD_VALUE: return "a value that is not UTF-8 or holds a NUL";
        case RL_CV_BAD_DIGEST: return "the values do not digest to the key";
        case RL_CV_BAD_DUPLICATE: return "the import names the key twice";
        default: return "unknown reason";
    }
}

// the engine's device and stream, and the matcher's image as it stands now
int bind_engine(rl_rls_dev* S, rl_engine* e, rl_matcher* m) {
    RlTableView v;
    const int r = rl_internal_view(e, &v);
    if (r) return fail(S, r, "%s", rl_last_error(e));
    S->device = v.device;
    S->stream = v.stream;
    return m ? refresh_image(S, m) : RL_OK;
}

}  // namespace

extern "C" {

int rl_rls_dev_plan(rl_rls_dev** st, rl_engine* e, rl_matcher* m, int method, uint64_t n, const uint8_t* buf,
                    const uint64_t* off, uint64_t now_us, uint64_t* out_n_store, uint64_t* out_n_ctr,
                    const RlsDevReq** out_req) {
    if (!st || !e || !m || !out_n_store || !out_n_ctr || !out_req) return RL_FATAL;
    if (!*st) *st = new rl_rls_dev();
    rl_rls_dev* S = *st;
    uint32_t per_req = 0;
    int r = stage_batch(S, e, m, n, buf, off, per_req);
    if (r) return r;
    RL_CUDA(S, S->h_req.grow(n + 1));
    RL_CUDA(S, S->d_req.grow(n + 1));
    RL_CUDA(S, S->d_count.grow(n + 1));
    RL_CUDA(S, S->d_start.grow(n + 1));
    RlsPlanArgs a;
    a.buf = S->d_buf.p;
    a.off = S->d_off.p;
    a.n = n;
    a.img = rl_img_view(S->image.data(), S->d_image.p);
    a.per_req = per_req;
    a.ent = S->d_ent.p;
    a.scratch = S->d_scratch.p;
    a.req = S->d_req.p;
    a.count = S->d_count.p;
    const uint32_t threads = 128;
    k_rls_plan<<<blocks_for(n + 1, threads), threads, 0, S->stream>>>(a);
    RL_CUDA(S, cudaGetLastError());
    size_t tmp = 0;
    RL_CUDA(S, cub::DeviceScan::ExclusiveSum(nullptr, tmp, S->d_count.p, S->d_start.p, (int64_t)(n + 1), S->stream));
    RL_CUDA(S, S->d_cub.grow(tmp + 1));
    RL_CUDA(S, cub::DeviceScan::ExclusiveSum(S->d_cub.p, tmp, S->d_count.p, S->d_start.p, (int64_t)(n + 1), S->stream));
    // the one read before the store call: how many store requests and counters the batch has
    if ((r = read_totals(S, S->h_total.p, S->d_start.p + n, sizeof(unsigned long long)))) return r;
    const uint64_t n_store = S->h_total.p[0] >> 32, n_ctr = S->h_total.p[0] & 0xFFFFFFFFull;
    if ((r = grow_csr(S, n_store, n_ctr))) return r;
    RlsScatterArgs b;
    b.req = S->d_req.p;
    b.scratch = S->d_scratch.p;
    b.start = S->d_start.p;
    b.n = n;
    b.per_req = per_req;
    b.method = method;
    b.now_us = now_us;
    b.ctr_off = S->d_ctr_off.p;
    b.ctrs = S->d_ctrs.p;
    b.delta = S->d_delta.p;
    b.now = S->d_now.p;
    k_rls_scatter<<<blocks_for(n + 1, threads), threads, 0, S->stream>>>(b);
    RL_CUDA(S, cudaGetLastError());
    if ((r = record_vars<CvWire>(S, e, 2, n, per_req, S->d_count.p, nullptr))) return r;
    return close_plan(S, n, n_store, n_ctr, S->h_req, S->d_req, out_n_store, out_n_ctr, out_req);
}

int rl_rls_dev_copy_plan(rl_rls_dev* S, uint32_t* ctr_off, rl_counter* ctrs, uint64_t* delta, uint8_t* load) {
    if (!S) return RL_FATAL;
    RL_CUDA(S, cudaSetDevice(S->device));
    RL_CUDA(S, cudaMemcpyAsync(ctr_off, S->d_ctr_off.p, (S->n_store + 1) * sizeof(uint32_t), cudaMemcpyDeviceToHost, S->stream));
    if (S->n_ctr) RL_CUDA(S, cudaMemcpyAsync(ctrs, S->d_ctrs.p, S->n_ctr * sizeof(rl_counter), cudaMemcpyDeviceToHost, S->stream));
    if (S->n_store) {
        RL_CUDA(S, cudaMemcpyAsync(delta, S->d_delta.p, S->n_store * sizeof(uint64_t), cudaMemcpyDeviceToHost, S->stream));
        if (load) RL_CUDA(S, cudaMemcpyAsync(load, S->d_load.p, S->n_store, cudaMemcpyDeviceToHost, S->stream));
    }
    RL_CUDA(S, cudaStreamSynchronize(S->stream));
    return RL_OK;
}

int rl_rls_dev_decide(rl_rls_dev* S, rl_engine* e, int method, int load_counters, uint8_t* limited, uint32_t* first_limited,
                      uint64_t* remaining, uint64_t* ttl_us, uint32_t* ctr_off, rl_counter* ctrs) {
    if (!S || !e) return RL_FATAL;
    if (S->n_store == 0) return RL_OK;
    RL_CUDA(S, cudaSetDevice(S->device));
    const StoreOp op = store_op(false, method);
    int st = reserve_outputs(S, load_counters != 0);
    if (st == RL_OK) st = store_call(S, e, op, 0, S->n_store, S->d_ctr_off.p, 0, load_counters != 0);
    if (st != RL_OK) return st;
    return copy_outputs(S, op != UPDATE, load_counters != 0, limited, first_limited, remaining, ttl_us, ctr_off, ctrs);
}

int rl_http_dev_plan(rl_rls_dev** st, rl_engine* e, rl_matcher* m, int endpoint, uint64_t n, const uint8_t* buf,
                     const uint64_t* off, uint64_t now_us, uint64_t* out_n_store, uint64_t* out_n_ctr,
                     const HttpDevReq** out_req, const HttpRun** out_runs, uint32_t* out_n_runs) {
    if (!st || !e || !m || !out_n_store || !out_n_ctr || !out_req || !out_runs || !out_n_runs) return RL_FATAL;
    if (!*st) *st = new rl_rls_dev();
    rl_rls_dev* S = *st;
    uint32_t per_req = 0;
    int r = stage_batch(S, e, m, n, buf, off, per_req);
    if (r) return r;
    const uint64_t bytes = n ? off[n] : 0;
    // the read before the store call: the head and up to kRunsRead store calls (a batch with more reads the rest after)
    const uint64_t kRunsRead = 1024;
    RL_CUDA(S, S->h_hreq.grow(n + 1));
    RL_CUDA(S, S->h_runs.grow(RL_HTTP_RUNS_HEAD + 3 * (n + 1)));
    RL_CUDA(S, S->d_txt.grow(bytes + 1));
    RL_CUDA(S, S->d_bits.grow(bytes / 8 + n + 1));
    RL_CUDA(S, S->d_hreq.grow(n + 1));
    RL_CUDA(S, S->d_hcount.grow(n + 1));
    RL_CUDA(S, S->d_hstart.grow(n + 1));
    RL_CUDA(S, S->d_runs.grow(RL_HTTP_RUNS_HEAD + 3 * (n + 1)));
    HttpPlanArgs a;
    a.buf = S->d_buf.p;
    a.off = S->d_off.p;
    a.n = n;
    a.img = rl_img_view(S->image.data(), S->d_image.p);
    a.per_req = per_req;
    a.endpoint = endpoint;
    a.txt = S->d_txt.p;
    a.bits = S->d_bits.p;
    a.ent = S->d_ent.p;
    a.scratch = S->d_scratch.p;
    a.req = S->d_hreq.p;
    a.count = S->d_hcount.p;
    const uint32_t threads = 128;
    k_http_plan<<<blocks_for(n + 1, threads), threads, 0, S->stream>>>(a);
    RL_CUDA(S, cudaGetLastError());
    size_t tmp = 0;
    const HttpScan zero{0, 0, 0, 0, 0, {0, 0}};
    RL_CUDA(S, cub::DeviceScan::ExclusiveScan(nullptr, tmp, S->d_hcount.p, S->d_hstart.p, HttpScanOp(), zero, (int64_t)(n + 1),
                                               S->stream));
    RL_CUDA(S, S->d_cub.grow(tmp + 1));
    RL_CUDA(S, cub::DeviceScan::ExclusiveScan(S->d_cub.p, tmp, S->d_hcount.p, S->d_hstart.p, HttpScanOp(), zero, (int64_t)(n + 1),
                                               S->stream));
    HttpRunsArgs ra{S->d_hcount.p, S->d_hstart.p, n, S->d_runs.p};
    k_http_runs<<<blocks_for(n + 1, threads), threads, 0, S->stream>>>(ra);
    RL_CUDA(S, cudaGetLastError());
    const uint64_t first_read = RL_HTTP_RUNS_HEAD + 3 * std::min<uint64_t>(n, kRunsRead);
    if ((r = read_totals(S, S->h_runs.p, S->d_runs.p, first_read * sizeof(uint32_t)))) return r;
    const uint64_t n_store = S->h_runs.p[0], n_ctr = S->h_runs.p[1], n_runs = S->h_runs.p[2];
    if (RL_HTTP_RUNS_HEAD + 3 * n_runs > first_read &&
        (r = read_totals(S, S->h_runs.p + first_read, S->d_runs.p + first_read,
                         (RL_HTTP_RUNS_HEAD + 3 * n_runs - first_read) * sizeof(uint32_t))))
        return r;
    if ((r = grow_csr(S, n_store, n_ctr))) return r;
    RL_CUDA(S, S->d_ctr_run.grow(n_store + n_runs + 1));
    RL_CUDA(S, S->d_load.grow(n_store + 1));
    HttpScatterArgs b;
    b.req = S->d_hreq.p;
    b.scratch = S->d_scratch.p;
    b.start = S->d_hstart.p;
    b.runs = S->d_runs.p + RL_HTTP_RUNS_HEAD;
    b.n = n;
    b.per_req = per_req;
    b.endpoint = endpoint;
    b.now_us = now_us;
    b.ctr_off = S->d_ctr_off.p;
    b.ctr_run = S->d_ctr_run.p;
    b.ctrs = S->d_ctrs.p;
    b.delta = S->d_delta.p;
    b.now = S->d_now.p;
    b.load = S->d_load.p;
    k_http_scatter<<<blocks_for(n + 1, threads), threads, 0, S->stream>>>(b);
    RL_CUDA(S, cudaGetLastError());
    if ((r = record_vars<CvJson>(S, e, 3, n, per_req, nullptr, S->d_hcount.p))) return r;
    if ((r = close_plan(S, n, n_store, n_ctr, S->h_hreq, S->d_hreq, out_n_store, out_n_ctr, out_req))) return r;
    S->n_runs = (uint32_t)n_runs;
    *out_runs = reinterpret_cast<const HttpRun*>(S->h_runs.p + RL_HTTP_RUNS_HEAD);
    *out_n_runs = (uint32_t)n_runs;
    return RL_OK;
}

int rl_http_dev_decide(rl_rls_dev* S, rl_engine* e, int endpoint, int* run_status, uint8_t* limited, uint32_t* first_limited,
                       uint64_t* remaining, uint64_t* ttl_us, uint32_t* ctr_off, rl_counter* ctrs) {
    if (!S || !e || !run_status) return RL_FATAL;
    if (S->n_store == 0) return RL_OK;
    RL_CUDA(S, cudaSetDevice(S->device));
    const StoreOp op = store_op(true, endpoint);
    const HttpRun* runs = reinterpret_cast<const HttpRun*>(S->h_runs.p + RL_HTTP_RUNS_HEAD);
    bool any_load = false;
    for (uint32_t k = 0; k < S->n_runs; k++) any_load = any_load || runs[k].load;
    int r = reserve_outputs(S, any_load);
    if (r) return r;
    // one store call per run, in batch order: run k's CSR starts at ctr_run[runs[k].store + k] and counts from 0
    for (uint32_t k = 0; k < S->n_runs; k++) {
        const HttpRun& R = runs[k];
        const uint64_t j1 = k + 1 < S->n_runs ? runs[k + 1].store : S->n_store;
        run_status[k] = store_call(S, e, op, R.store, j1 - R.store, S->d_ctr_run.p + R.store + k, R.ctr, R.load != 0);
    }
    return copy_outputs(S, op != UPDATE, any_load, limited, first_limited, remaining, ttl_us, ctr_off, ctrs);
}

int rl_rls_dev_shard_send(rl_rls_dev* S, rl_shard_batch* sb, int empty, int http, int method, int load_counters, int* out_failed) {
    if (!sb || !out_failed) return RL_FATAL;
    *out_failed = RL_OK;
    const int op = store_op(http != 0, method);
    if (!empty && S && S->n_store) {
        RL_CUDA(S, cudaSetDevice(S->device));
        const int r = reserve_outputs(S, load_counters != 0);
        if (r == RL_OK)
            return rl_shard_batch_send(sb, S->n_store, S->n_ctr, S->d_ctr_off.p, S->d_ctrs.p, S->d_delta.p, S->d_now.p, op,
                                       http ? S->d_load.p : nullptr, http ? 0 : load_counters);
        *out_failed = r;  // the step still goes out, empty: no peer waits for it
    }
    return rl_shard_batch_send(sb, 0, 0, nullptr, nullptr, nullptr, nullptr, op, nullptr, 0);
}

int rl_rls_dev_shard_collect(rl_rls_dev* S, rl_shard_batch* sb, int load_counters, uint8_t* limited, uint32_t* first_limited,
                             uint64_t* remaining, uint64_t* ttl_us, uint32_t* ctr_off, rl_counter* ctrs) {
    if (!sb) return RL_FATAL;
    const bool any = S && S->n_store;
    const bool lc = any && load_counters;
    const int st = rl_shard_batch_collect(sb, any ? S->d_lim.p : nullptr, any ? S->d_first.p : nullptr, lc ? S->d_rem.p : nullptr,
                                          lc ? S->d_ttl.p : nullptr);
    if (!any) return st;
    const int r = copy_outputs(S, true, lc, limited, first_limited, remaining, ttl_us, ctr_off, ctrs);
    if (r) return r;
    RL_CUDA(S, cudaStreamSynchronize(S->stream));
    return st;
}

int rl_rls_dev_wait(rl_rls_dev* S) {
    if (!S) return RL_FATAL;
    RL_CUDA(S, cudaSetDevice(S->device));
    RL_CUDA(S, cudaStreamSynchronize(S->stream));
    return RL_OK;
}

int rl_cv_dev_configure(rl_rls_dev** st, rl_engine* e, uint64_t max_keys, uint64_t arena_bytes) {
    if (!st || !e) return RL_FATAL;
    if (!*st) *st = new rl_rls_dev();
    rl_rls_dev* S = *st;
    int r = bind_engine(S, e, nullptr);
    if (r) return r;
    RL_CUDA(S, cudaStreamSynchronize(S->stream));  // no batch may still write the old dictionary
    S->cv_slots = S->cv_arena_bytes = 0;
    S->cv_full_next = true;
    RL_CUDA(S, S->d_cv_slots.exact(0));
    RL_CUDA(S, S->d_cv_arena.exact(0));
    RL_CUDA(S, S->d_cv_ctl.exact(0));
    if (max_keys == 0 && arena_bytes == 0) return RL_OK;
    if (max_keys == 0 || arena_bytes == 0 || max_keys > (1ull << 40))
        return fail(S, RL_FATAL, "keeping counter variables needs max_keys in [1, 2^40] and arena_bytes > 0");
    uint64_t slots = 16;
    while (slots < max_keys) slots *= 2;
    RL_CUDA(S, S->d_cv_slots.exact(slots));
    RL_CUDA(S, S->d_cv_arena.exact(arena_bytes));
    RL_CUDA(S, S->d_cv_ctl.exact(RL_CV_CTL_WORDS));
    RL_CUDA(S, cudaMemsetAsync(S->d_cv_slots.p, 0, slots * sizeof(CvSlot), S->stream));
    RL_CUDA(S, cudaMemsetAsync(S->d_cv_ctl.p, 0, RL_CV_CTL_WORDS * sizeof(unsigned long long), S->stream));
    RL_CUDA(S, cudaStreamSynchronize(S->stream));
    S->cv_slots = slots;
    S->cv_arena_bytes = arena_bytes;
    return RL_OK;
}

int rl_cv_dev_stats(rl_rls_dev* S, uint64_t* out_slots, uint64_t* out_keys, uint64_t* out_arena_used, uint64_t* out_dropped) {
    uint64_t w[RL_CV_CTL_WORDS] = {0, 0, 0, 0};
    if (S && S->cv_slots) {
        RL_CUDA(S, cudaSetDevice(S->device));
        RL_CUDA(S, cudaMemcpyAsync(w, S->d_cv_ctl.p, sizeof w, cudaMemcpyDeviceToHost, S->stream));
        RL_CUDA(S, cudaStreamSynchronize(S->stream));
    }
    if (out_slots) *out_slots = S ? S->cv_slots : 0;
    if (out_keys) *out_keys = w[RL_CV_KEYS];
    if (out_arena_used) *out_arena_used = S ? std::min<uint64_t>(w[RL_CV_CURSOR], S->cv_arena_bytes) : 0;
    if (out_dropped) *out_dropped = w[RL_CV_DROPPED];
    return RL_OK;
}

int rl_cv_dev_lookup(rl_rls_dev** st, rl_engine* e, rl_matcher* m, uint64_t n, const uint32_t* limit_id, const uint64_t* key_lo,
                     const uint64_t* key_hi, const uint8_t** out_blobs, const uint64_t** out_blob_off, const uint8_t** out_unnamed) {
    if (!st || !e || !m || (n && (!limit_id || !key_lo || !key_hi)) || !out_blobs || !out_blob_off || !out_unnamed) return RL_FATAL;
    if (!*st) *st = new rl_rls_dev();
    rl_rls_dev* S = *st;
    int r = bind_engine(S, e, m);
    if (r) return r;
    S->h_cv_pos.assign(n + 1, 0);
    S->h_cv_src.assign(n + 1, 0);
    S->h_cv_unnamed.assign(n + 1, 0);
    S->h_cv_out.assign(1, 0);
    if (!S->cv_slots) {  // keeping is off: every qualified counter is unnamed
        const RlImage I = rl_img_view(S->image.data(), S->image.data());
        for (uint64_t i = 0; i < n; i++) S->h_cv_unnamed[i] = limit_id[i] < I.n_limits && I.lims[5ull * limit_id[i] + 4] != 0;
    } else if (n) {
        RL_CUDA(S, S->d_cv_lid.grow(n));
        RL_CUDA(S, S->d_cv_lo.grow(n));
        RL_CUDA(S, S->d_cv_hi.grow(n));
        RL_CUDA(S, S->d_cv_src.grow(n));
        RL_CUDA(S, S->d_cv_len.grow(n + 1));
        RL_CUDA(S, S->d_cv_pos.grow(n + 1));
        RL_CUDA(S, cudaMemcpyAsync(S->d_cv_lid.p, limit_id, n * sizeof(uint32_t), cudaMemcpyHostToDevice, S->stream));
        RL_CUDA(S, cudaMemcpyAsync(S->d_cv_lo.p, key_lo, n * sizeof(uint64_t), cudaMemcpyHostToDevice, S->stream));
        RL_CUDA(S, cudaMemcpyAsync(S->d_cv_hi.p, key_hi, n * sizeof(uint64_t), cudaMemcpyHostToDevice, S->stream));
        CvLookupArgs a{S->d_cv_lid.p, S->d_cv_lo.p, S->d_cv_hi.p, n, rl_img_view(S->image.data(), S->d_image.p), cv_dict(S),
                       S->d_cv_len.p, S->d_cv_src.p};
        const uint32_t threads = 256;
        k_counter_vars_lookup<<<blocks_for(n + 1, threads), threads, 0, S->stream>>>(a);
        RL_CUDA(S, cudaGetLastError());
        size_t tmp = 0;
        RL_CUDA(S, cub::DeviceScan::ExclusiveSum(nullptr, tmp, S->d_cv_len.p, S->d_cv_pos.p, (int64_t)(n + 1), S->stream));
        RL_CUDA(S, S->d_cub.grow(tmp + 1));
        RL_CUDA(S, cub::DeviceScan::ExclusiveSum(S->d_cub.p, tmp, S->d_cv_len.p, S->d_cv_pos.p, (int64_t)(n + 1), S->stream));
        unsigned long long total = 0;
        RL_CUDA(S, cudaMemcpyAsync(&total, S->d_cv_pos.p + n, sizeof total, cudaMemcpyDeviceToHost, S->stream));
        RL_CUDA(S, cudaStreamSynchronize(S->stream));
        RL_CUDA(S, S->d_cv_out.grow(total + 1));
        CvGatherArgs g{S->d_cv_pos.p, S->d_cv_len.p, S->d_cv_src.p, n, S->d_cv_arena.p, S->d_cv_out.p};
        k_counter_vars_gather<<<blocks_for(n, threads), threads, 0, S->stream>>>(g);
        RL_CUDA(S, cudaGetLastError());
        rl_internal_launched(e, 2);
        S->h_cv_out.resize(total + 1);
        if (total) RL_CUDA(S, cudaMemcpyAsync(S->h_cv_out.data(), S->d_cv_out.p, total, cudaMemcpyDeviceToHost, S->stream));
        RL_CUDA(S, cudaMemcpyAsync(S->h_cv_pos.data(), S->d_cv_pos.p, (n + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, S->stream));
        RL_CUDA(S, cudaMemcpyAsync(S->h_cv_src.data(), S->d_cv_src.p, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, S->stream));
        RL_CUDA(S, cudaStreamSynchronize(S->stream));
        for (uint64_t i = 0; i < n; i++) S->h_cv_unnamed[i] = S->h_cv_src[i] == RL_CV_NONE;
    }
    *out_blobs = S->h_cv_out.data();
    *out_blob_off = reinterpret_cast<const uint64_t*>(S->h_cv_pos.data());
    *out_unnamed = S->h_cv_unnamed.data();
    return RL_OK;
}

int rl_cv_dev_gc(rl_rls_dev** st, rl_engine* e, rl_matcher* m, uint64_t now_us, uint64_t* out_kept, uint64_t* out_freed) {
    if (!st || !e || !m) return RL_FATAL;
    if (out_kept) *out_kept = 0;
    if (out_freed) *out_freed = 0;
    if (!*st || !(*st)->cv_slots) return RL_OK;
    rl_rls_dev* S = *st;
    int r = bind_engine(S, e, m);
    if (r) return r;
    uint64_t before[RL_CV_CTL_WORDS];
    RL_CUDA(S, cudaMemcpyAsync(before, S->d_cv_ctl.p, sizeof before, cudaMemcpyDeviceToHost, S->stream));
    // mark what the engine's live counters reference, then copy it into a fresh table and arena
    uint32_t launched = 0;
    if ((r = mark_live(S, e, nullptr, 0, now_us, launched))) return r;
    if ((r = kept_positions(S))) return r;
    DevBuf<CvSlot> slots2;
    DevBuf<uint8_t> arena2;
    DevBuf<unsigned long long> ctl2;
    if ((r = rebuild_fresh(S, slots2, arena2, ctl2))) return r;
    rl_internal_launched(e, launched + 2);
    RL_CUDA(S, cudaStreamSynchronize(S->stream));  // the old dictionary is read until here
    S->d_cv_slots.swap(slots2);
    S->d_cv_arena.swap(arena2);
    S->d_cv_ctl.swap(ctl2);
    S->cv_full_next = true;
    uint64_t after[RL_CV_CTL_WORDS];
    RL_CUDA(S, cudaMemcpy(after, S->d_cv_ctl.p, sizeof after, cudaMemcpyDeviceToHost));
    if (out_kept) *out_kept = after[RL_CV_KEYS];
    if (out_freed) *out_freed = before[RL_CV_KEYS] - std::min(before[RL_CV_KEYS], after[RL_CV_KEYS]);
    return RL_OK;
}

int rl_cv_dev_export(rl_rls_dev** st, rl_engine* e, rl_matcher* m, const uint32_t* ns_ids, uint32_t n_ns, uint64_t now_us,
                     uint64_t cap, uint64_t bytes_cap, uint32_t* out_varset, uint64_t* out_key_lo, uint64_t* out_key_hi,
                     uint64_t* out_blob_off, uint8_t* out_blobs, uint64_t* out_count, uint64_t* out_bytes) {
    if (!st || !e || !m || !out_count || !out_bytes) return RL_FATAL;
    *out_count = *out_bytes = 0;
    if (!*st || !(*st)->cv_slots) return RL_OK;
    rl_rls_dev* S = *st;
    int r = bind_engine(S, e, m);
    if (r) return r;
    uint32_t launched = 0;
    if ((r = mark_live(S, e, ns_ids, n_ns, now_us, launched))) return r;
    rl_internal_launched(e, launched);
    return export_marked(S, e, cap, bytes_cap, out_varset, out_key_lo, out_key_hi, out_blob_off, out_blobs, out_count, out_bytes);
}

int rl_cv_dev_drain(rl_rls_dev** st, rl_engine* e, rl_matcher* m, uint64_t cap, uint64_t bytes_cap, uint32_t* out_varset,
                    uint64_t* out_key_lo, uint64_t* out_key_hi, uint64_t* out_blob_off, uint8_t* out_blobs, uint64_t* out_count,
                    uint64_t* out_bytes, int* out_full) {
    if (!st || !e || !m || !out_count || !out_bytes || !out_full) return RL_FATAL;
    *out_count = *out_bytes = 0;
    *out_full = 0;
    if (!*st || !(*st)->cv_slots) return RL_OK;
    rl_rls_dev* S = *st;
    int r = bind_engine(S, e, m);
    if (r) return r;
    unsigned long long cursor = 0;
    RL_CUDA(S, cudaMemcpyAsync(&cursor, S->d_cv_ctl.p + RL_CV_CURSOR, sizeof cursor, cudaMemcpyDeviceToHost, S->stream));
    RL_CUDA(S, cudaStreamSynchronize(S->stream));
    if (S->cv_full_next) {  // the caller takes a full export; the next drain starts from here
        *out_full = 1;
        S->cv_since = cursor;
        S->cv_full_next = false;
        return RL_OK;
    }
    const uint64_t slots = S->cv_slots;
    RL_CUDA(S, S->d_cv_mark.grow(slots + 1));
    RL_CUDA(S, S->d_cv_len.grow(slots + 1));
    RL_CUDA(S, S->d_cv_pos.grow(slots + 1));
    RL_CUDA(S, cudaMemsetAsync(S->d_cv_mark.p + slots, 0, 1, S->stream));
    k_counter_vars_since<<<blocks_for(slots, 256), 256, 0, S->stream>>>(cv_dict(S), S->cv_since, S->d_cv_mark.p);
    RL_CUDA(S, cudaGetLastError());
    rl_internal_launched(e, 1);
    if ((r = export_marked(S, e, cap, bytes_cap, out_varset, out_key_lo, out_key_hi, out_blob_off, out_blobs, out_count, out_bytes)))
        return r;
    if (*out_count <= cap && *out_bytes <= bytes_cap) S->cv_since = cursor;  // consumed only when it was handed over
    return RL_OK;
}

int rl_cv_dev_import(rl_rls_dev** st, rl_engine* e, rl_matcher* m, uint64_t n, const uint32_t* varset, const uint64_t* key_lo,
                     const uint64_t* key_hi, const uint64_t* blob_off, const uint8_t* blobs, uint64_t* out_added) {
    if (!st || !e || !m || (n && (!varset || !key_lo || !key_hi || !blob_off))) return RL_FATAL;
    if (out_added) *out_added = 0;
    if (!*st) *st = new rl_rls_dev();
    rl_rls_dev* S = *st;
    if (!S->cv_slots) return fail(S, RL_FATAL, "importing counter variables needs keeping on (rl_rls_keep_counter_vars)");
    if (n == 0) return RL_OK;
    for (uint64_t i = 0; i < n; i++)
        if (blob_off[i + 1] < blob_off[i])
            return fail(S, RL_FATAL, "counter variable entry %llu refused: blob_off decreases after it", (unsigned long long)i);
    const uint64_t bytes = blob_off[n];
    if (bytes && !blobs) return fail(S, RL_FATAL, "importing counter variables: blobs is NULL");
    int r = bind_engine(S, e, m);
    if (r) return r;
    // varset -> (first variable, variables) of the image's qualified limits
    const RlImage H = rl_img_view(S->image.data(), S->image.data());
    uint32_t n_vs = 1;
    for (uint32_t l = 0; l < H.n_limits; l++) n_vs = std::max(n_vs, H.lims[5ull * l + 4] + 1);
    std::vector<uint32_t> vs_vars(2ull * n_vs, 0);
    for (uint32_t l = 0; l < H.n_limits; l++) {
        const uint32_t* L = H.lims + 5ull * l;
        if (L[4] && L[3]) {
            vs_vars[2ull * L[4]] = L[2];
            vs_vars[2ull * L[4] + 1] = L[3];
        }
    }
    In<uint32_t> d_vs, d_vt;
    In<uint64_t> d_lo, d_hi, d_off;
    In<uint8_t> d_blobs;
    RL_CUDA(S, d_vs.set(varset, n, RL_MEM_HOST, S->stream));
    RL_CUDA(S, d_lo.set(key_lo, n, RL_MEM_HOST, S->stream));
    RL_CUDA(S, d_hi.set(key_hi, n, RL_MEM_HOST, S->stream));
    RL_CUDA(S, d_off.set(blob_off, n + 1, RL_MEM_HOST, S->stream));
    RL_CUDA(S, d_blobs.set(blobs, bytes, RL_MEM_HOST, S->stream));
    RL_CUDA(S, d_vt.set(vs_vars.data(), vs_vars.size(), RL_MEM_HOST, S->stream));
    DevBuf<unsigned long long> len, pos, bad;
    RL_CUDA(S, len.exact(n + 1));
    RL_CUDA(S, pos.exact(n + 1));
    RL_CUDA(S, bad.exact(1));
    RL_CUDA(S, cudaMemsetAsync(bad.p, 0xFF, sizeof(unsigned long long), S->stream));
    CvImportArgs a{d_vs.p, d_lo.p, d_hi.p, d_off.p, d_blobs.p, n, rl_img_view(S->image.data(), S->d_image.p), d_vt.p, n_vs,
                   cv_dict(S), len.p, pos.p, 0, bad.p};
    // check every entry against the image and the dictionary; each new blob's position after the kept ones
    const uint32_t threads = 128;
    k_counter_vars_check<<<blocks_for(n + 1, threads), threads, 0, S->stream>>>(a);
    RL_CUDA(S, cudaGetLastError());
    size_t tmp = 0;
    RL_CUDA(S, cub::DeviceScan::ExclusiveSum(nullptr, tmp, len.p, pos.p, (int64_t)(n + 1), S->stream));
    RL_CUDA(S, S->d_cub.grow(tmp + 1));
    RL_CUDA(S, cub::DeviceScan::ExclusiveSum(S->d_cub.p, tmp, len.p, pos.p, (int64_t)(n + 1), S->stream));
    // every entry the dictionary holds, in a compacted arena
    const uint64_t slots = S->cv_slots;
    RL_CUDA(S, S->d_cv_mark.grow(slots + 1));
    RL_CUDA(S, S->d_cv_len.grow(slots + 1));
    RL_CUDA(S, S->d_cv_pos.grow(slots + 1));
    k_counter_vars_occupied<<<blocks_for(slots, 256), 256, 0, S->stream>>>(cv_dict(S), S->d_cv_mark.p);
    RL_CUDA(S, cudaGetLastError());
    if ((r = kept_positions(S))) return r;
    rl_internal_launched(e, 3);
    uint64_t before[RL_CV_CTL_WORDS];
    unsigned long long tot[3];  // bad, the new bytes, the kept bytes
    RL_CUDA(S, cudaMemcpyAsync(before, S->d_cv_ctl.p, sizeof before, cudaMemcpyDeviceToHost, S->stream));
    RL_CUDA(S, cudaMemcpyAsync(&tot[0], bad.p, sizeof tot[0], cudaMemcpyDeviceToHost, S->stream));
    RL_CUDA(S, cudaMemcpyAsync(&tot[1], pos.p + n, sizeof tot[1], cudaMemcpyDeviceToHost, S->stream));
    RL_CUDA(S, cudaMemcpyAsync(&tot[2], S->d_cv_pos.p + slots, sizeof tot[2], cudaMemcpyDeviceToHost, S->stream));
    RL_CUDA(S, cudaStreamSynchronize(S->stream));
    if (tot[0] != RL_CV_GOOD) return fail(S, RL_FATAL, "counter variable entry %llu refused: %s", tot[0] >> 8, cv_reason(tot[0] & 0xFF));
    if (tot[1] == 0) return RL_OK;  // every key is held already
    if (tot[1] + tot[2] > S->cv_arena_bytes)
        return fail(S, RL_TRANSIENT, "the dictionary's arena has no room: %llu bytes kept + %llu imported > %llu", tot[2], tot[1],
                    (unsigned long long)S->cv_arena_bytes);
    // commit: a fresh table with every entry, then the new ones; swapped in only if each found its slot
    DevBuf<CvSlot> slots2;
    DevBuf<uint8_t> arena2;
    DevBuf<unsigned long long> ctl2;
    if ((r = rebuild_fresh(S, slots2, arena2, ctl2))) return r;
    a.dict = CvDict{slots2.p, slots - 1, arena2.p, S->cv_arena_bytes, ctl2.p};
    a.base = tot[2];
    k_counter_vars_import<<<blocks_for(n + 1, threads), threads, 0, S->stream>>>(a);
    RL_CUDA(S, cudaGetLastError());
    rl_internal_launched(e, 2);
    uint64_t after[RL_CV_CTL_WORDS];
    RL_CUDA(S, cudaMemcpyAsync(after, ctl2.p, sizeof after, cudaMemcpyDeviceToHost, S->stream));
    RL_CUDA(S, cudaMemcpyAsync(&tot[0], bad.p, sizeof tot[0], cudaMemcpyDeviceToHost, S->stream));
    RL_CUDA(S, cudaStreamSynchronize(S->stream));
    if (tot[0] != RL_CV_GOOD) {  // which thread saw the other's slot depends on the schedule: name the later entry
        std::unordered_map<uint64_t, uint64_t> seen;  // (a hash of) the key -> first entry
        for (uint64_t i = 0; i < n; i++) {
            const uint64_t h = rl_cv_fp(varset[i], key_lo[i], key_hi[i]);
            auto it = seen.find(h);
            if (it != seen.end() && varset[it->second] == varset[i] && key_lo[it->second] == key_lo[i] && key_hi[it->second] == key_hi[i])
                return fail(S, RL_FATAL, "counter variable entry %llu refused: %s (entry %llu)", (unsigned long long)i,
                            cv_reason(RL_CV_BAD_DUPLICATE), (unsigned long long)it->second);
            seen.emplace(h, i);
        }
        return fail(S, RL_FATAL, "counter variable entry %llu refused: %s", tot[0] >> 8, cv_reason(tot[0] & 0xFF));
    }
    if (after[RL_CV_DROPPED] != before[RL_CV_DROPPED])
        return fail(S, RL_TRANSIENT, "the dictionary has no room: %llu entries found no free slot within %u probes",
                    (unsigned long long)(after[RL_CV_DROPPED] - before[RL_CV_DROPPED]), RL_CV_PROBE);
    S->d_cv_slots.swap(slots2);
    S->d_cv_arena.swap(arena2);
    S->d_cv_ctl.swap(ctl2);
    S->cv_full_next = true;
    if (out_added) *out_added = after[RL_CV_KEYS] - before[RL_CV_KEYS];
    return RL_OK;
}

const char* rl_rls_dev_error(rl_rls_dev* S) { return S ? S->err.c_str() : "no device plan state"; }

void rl_rls_dev_destroy(rl_rls_dev* S) {
    if (!S) return;
    cudaSetDevice(S->device);
    if (S->stream) cudaStreamSynchronize(S->stream);
    delete S;
}

}  // extern "C"
