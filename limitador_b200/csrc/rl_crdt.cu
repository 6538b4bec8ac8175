// rl_crdt.cu — host side of the replicated counter value (include/rl_crdt.h): table, staging, launches.
#include <cuda_runtime.h>

#include <cstring>
#include <string>
#include <vector>

#include "rl_crdt.cuh"
#include "rl_cuda_host.h"

struct rl_crdt {
    int device = 0;
    cudaStream_t stream = nullptr;
    DevBuf<uint8_t> d_rows;
    DevBuf<uint32_t> d_err;
    uint64_t capacity = 0;
    uint32_t actors = 1, actors_pad = 2, self_actor = 0, row_bytes = 48;
    uint64_t launches = 0;
    std::string last_error;
};

namespace {

template <class... A>
int fail(rl_crdt* c, int status, const char* fmt, A... a) {
    if (c) c->last_error = rl_format(fmt, a...);
    return status;
}

RlCrdtTab tab_of(const rl_crdt* c) {
    RlCrdtTab T;
    T.rows = c->d_rows.p;
    T.mask = c->capacity - 1;
    T.row_bytes = c->row_bytes;
    T.actors = c->actors;
    T.actors_pad = c->actors_pad;
    T.self_actor = c->self_actor;
    T.err = c->d_err.p;
    return T;
}

// Wait for the call's kernels and translate the sticky device error.
int finish(rl_crdt* c) {
    uint32_t code = 0;
    RL_CUDA(c, cudaMemcpyAsync(&code, c->d_err.p, sizeof code, cudaMemcpyDeviceToHost, c->stream));
    RL_CUDA(c, cudaStreamSynchronize(c->stream));
    if (code == 0) return RL_OK;
    RL_CUDA(c, cudaMemset(c->d_err.p, 0, sizeof(uint32_t)));
    switch (code) {
        case 1: return fail(c, RL_TRANSIENT, "replicated counter table full (capacity_rows=%llu): batch partially applied", (unsigned long long)c->capacity);
        case 2: return fail(c, RL_FATAL, "actor index out of range (actors=%u)", c->actors);
        case 3: return fail(c, RL_FATAL, "counter key must be non-zero with hi != ~0");
        default: return fail(c, RL_FATAL, "an update's value range lies outside the values array");
    }
}

uint32_t blocks_for(uint64_t n) { return (uint32_t)((n + 255) / 256); }

}  // namespace

extern "C" {

int rl_crdt_create(const rl_crdt_config* cfg, rl_crdt** out) {
    if (!cfg || !out || cfg->struct_size != sizeof(rl_crdt_config)) return RL_FATAL;
    *out = nullptr;
    if (cfg->actors < 1 || cfg->actors > RL_CRDT_MAX_ACTORS || cfg->self_actor >= cfg->actors || cfg->capacity_rows == 0 ||
        cfg->capacity_rows > (1ull << 32))
        return RL_FATAL;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || cfg->device < 0 || cfg->device >= ndev) {
        cudaGetLastError();
        return RL_FATAL;  // no CUDA device: there is no CPU implementation to fall back to
    }
    rl_crdt* c = new rl_crdt();
    c->device = cfg->device;
    c->actors = cfg->actors;
    c->actors_pad = (cfg->actors + 1u) & ~1u;
    c->self_actor = cfg->self_actor;
    c->row_bytes = 32 + 8 * c->actors_pad;
    c->capacity = 1;
    while (c->capacity < cfg->capacity_rows) c->capacity <<= 1;
    *out = c;  // handed out even on failure below so that the caller can read the error, then destroy
    RL_CUDA(c, cudaSetDevice(c->device));
    RL_CUDA(c, cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    RL_CUDA(c, c->d_rows.exact(c->capacity * c->row_bytes));
    RL_CUDA(c, c->d_err.exact(1));
    RL_CUDA(c, cudaMemsetAsync(c->d_rows.p, 0, c->capacity * c->row_bytes, c->stream));
    RL_CUDA(c, cudaMemsetAsync(c->d_err.p, 0, sizeof(uint32_t), c->stream));
    RL_CUDA(c, cudaStreamSynchronize(c->stream));
    return RL_OK;
}

void rl_crdt_destroy(rl_crdt* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    if (c->stream) cudaStreamDestroy(c->stream);
    delete c;  // frees the device arrays, on the device made current above
}

const char* rl_crdt_last_error(rl_crdt* c) { return c ? c->last_error.c_str() : "null handle"; }
uint64_t rl_crdt_kernel_launches(rl_crdt* c) { return c ? c->launches : 0; }

int rl_crdt_inc(rl_crdt* c, uint64_t n, const rl_crdt_key* keys, const uint32_t* actor, const uint64_t* increment,
                const uint64_t* window_us, uint64_t now_us, int mem) {
    if (!c || n > 0xFFFFFFFFull || (n && (!keys || !actor || !increment || !window_us))) return fail(c, RL_FATAL, "rl_crdt_inc: bad arguments");
    if (n == 0) return RL_OK;
    RL_CUDA(c, cudaSetDevice(c->device));
    In<rl_crdt_key> k;
    In<uint32_t> a;
    In<uint64_t> inc, win;
    RL_CUDA(c, k.set(keys, n, mem, c->stream));
    RL_CUDA(c, a.set(actor, n, mem, c->stream));
    RL_CUDA(c, inc.set(increment, n, mem, c->stream));
    RL_CUDA(c, win.set(window_us, n, mem, c->stream));
    k_crdt_inc<<<blocks_for(n), 256, 0, c->stream>>>(tab_of(c), (uint32_t)n, k.p, a.p, inc.p, win.p, now_us);
    RL_CUDA(c, cudaGetLastError());
    c->launches++;
    return finish(c);
}

int rl_crdt_merge(rl_crdt* c, uint64_t n, const rl_crdt_update* updates, const uint32_t* actors, const uint64_t* values,
                  uint64_t n_values, uint64_t now_us, int mem) {
    if (!c || n > 0xFFFFFFFFull || (n && !updates) || (n_values && (!actors || !values))) return fail(c, RL_FATAL, "rl_crdt_merge: bad arguments");
    if (n == 0) return RL_OK;
    RL_CUDA(c, cudaSetDevice(c->device));
    In<rl_crdt_update> u;
    In<uint32_t> a;
    In<uint64_t> v;
    RL_CUDA(c, u.set(updates, n, mem, c->stream));
    RL_CUDA(c, a.set(actors, n_values, mem, c->stream));
    RL_CUDA(c, v.set(values, n_values, mem, c->stream));
    DevBuf<unsigned long long> row_of;
    RL_CUDA(c, row_of.alloc(n));
    // two launches: every reset (expiry + zeroed values) is complete before any value is merged
    k_crdt_merge_expiry<<<blocks_for(n), 256, 0, c->stream>>>(tab_of(c), (uint32_t)n, u.p, now_us, row_of.p);
    k_crdt_merge_values<<<blocks_for(n), 256, 0, c->stream>>>(tab_of(c), (uint32_t)n, u.p, a.p, v.p, n_values, row_of.p);
    RL_CUDA(c, cudaGetLastError());
    c->launches += 2;
    return finish(c);  // synchronises the stream before the scratch and the staged inputs are freed
}

int rl_crdt_read(rl_crdt* c, uint64_t n, const rl_crdt_key* keys, uint64_t now_us, int mem, uint64_t* out_value,
                 uint64_t* out_expiry_us) {
    if (!c || n > 0xFFFFFFFFull || (n && (!keys || !out_value))) return fail(c, RL_FATAL, "rl_crdt_read: bad arguments");
    if (n == 0) return RL_OK;
    RL_CUDA(c, cudaSetDevice(c->device));
    In<rl_crdt_key> k;
    RL_CUDA(c, k.set(keys, n, mem, c->stream));
    DevBuf<uint64_t> own_val, own_exp;
    uint64_t *d_val = out_value, *d_exp = out_expiry_us;
    if (mem != RL_MEM_DEVICE) {
        RL_CUDA(c, own_val.alloc(n));
        d_val = own_val.p;
        if (out_expiry_us) {
            RL_CUDA(c, own_exp.alloc(n));
            d_exp = own_exp.p;
        }
    }
    k_crdt_read<<<blocks_for(n), 256, 0, c->stream>>>(tab_of(c), (uint32_t)n, k.p, now_us, d_val, d_exp);
    RL_CUDA(c, cudaGetLastError());
    c->launches++;
    if (mem != RL_MEM_DEVICE) {
        RL_CUDA(c, cudaMemcpyAsync(out_value, own_val.p, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream));
        if (out_expiry_us) RL_CUDA(c, cudaMemcpyAsync(out_expiry_us, own_exp.p, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, c->stream));
    }
    return finish(c);
}

static int scan(rl_crdt* c, int mode, uint64_t now_us, uint64_t cap, rl_crdt_key* out_keys, uint64_t* out_a,
                uint64_t* out_expiry_us, uint64_t* out_values, uint64_t* out_count) {
    if (!c || (cap && (!out_keys || !out_expiry_us))) return fail(c, RL_FATAL, "scan: bad arguments");
    RL_CUDA(c, cudaSetDevice(c->device));
    const uint64_t dcap = cap ? cap : 1;
    DevBuf<rl_crdt_key> keys;
    DevBuf<uint64_t> a, exp, vals;
    DevBuf<unsigned long long> cnt_d;
    RL_CUDA(c, keys.alloc(dcap));
    RL_CUDA(c, a.alloc(dcap));
    RL_CUDA(c, exp.alloc(dcap));
    RL_CUDA(c, vals.alloc(dcap * c->actors));
    RL_CUDA(c, cnt_d.alloc(1));
    RL_CUDA(c, cudaMemsetAsync(cnt_d.p, 0, sizeof(unsigned long long), c->stream));
    k_crdt_scan<<<blocks_for(c->capacity), 256, 0, c->stream>>>(tab_of(c), mode, now_us, cap, keys.p, a.p, exp.p, vals.p, cnt_d.p);
    RL_CUDA(c, cudaGetLastError());
    c->launches++;
    unsigned long long cnt = 0;
    RL_CUDA(c, cudaMemcpyAsync(&cnt, cnt_d.p, sizeof cnt, cudaMemcpyDeviceToHost, c->stream));
    const int r = finish(c);
    if (r) return r;
    const uint64_t got = cnt < cap ? cnt : cap;
    if (got) {
        RL_CUDA(c, cudaMemcpy(out_keys, keys.p, got * sizeof(rl_crdt_key), cudaMemcpyDeviceToHost));
        RL_CUDA(c, cudaMemcpy(out_expiry_us, exp.p, got * sizeof(uint64_t), cudaMemcpyDeviceToHost));
        if (mode == 0 && out_a) RL_CUDA(c, cudaMemcpy(out_a, a.p, got * sizeof(uint64_t), cudaMemcpyDeviceToHost));
        if (mode == 1 && out_values) RL_CUDA(c, cudaMemcpy(out_values, vals.p, got * c->actors * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    }
    if (out_count) *out_count = cnt;
    return RL_OK;
}

int rl_crdt_clear(rl_crdt* c) {
    if (!c) return RL_FATAL;
    RL_CUDA(c, cudaSetDevice(c->device));
    RL_CUDA(c, cudaMemsetAsync(c->d_rows.p, 0, c->capacity * c->row_bytes, c->stream));
    RL_CUDA(c, cudaStreamSynchronize(c->stream));
    return RL_OK;
}

int rl_crdt_export(rl_crdt* c, uint64_t now_us, uint64_t cap, rl_crdt_key* out_keys, uint64_t* out_value,
                   uint64_t* out_expiry_us, uint64_t* out_count) {
    if (cap && !out_value) return fail(c, RL_FATAL, "rl_crdt_export: bad arguments");
    return scan(c, 0, now_us, cap, out_keys, out_value, out_expiry_us, nullptr, out_count);
}

int rl_crdt_dump(rl_crdt* c, uint64_t cap, rl_crdt_key* out_keys, uint64_t* out_expiry_us, uint64_t* out_values,
                 uint64_t* out_count) {
    if (cap && !out_values) return fail(c, RL_FATAL, "rl_crdt_dump: bad arguments");
    return scan(c, 1, 0, cap, out_keys, nullptr, out_expiry_us, out_values, out_count);
}

}  // extern "C"
