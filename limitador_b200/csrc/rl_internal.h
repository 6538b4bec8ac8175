// rl_internal.h — what the maintenance translation unit (rl_maint.cu) may see of an engine (rl_engine.cu owns the struct).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/rl_engine.h"
#include "rl_core.h"

struct RlTableView {
    uint8_t* rows;
    uint32_t cells, log2P, log2R, row_bytes;
    uint64_t capacity;  // rows
    uint32_t ns_cap, limits_cap;
    const RlLimitDev* limits;  // [limits_cap] device limit table: group (0 = not registered), cell, qualified
    const RlCellDesc* desc;    // [row groups][8] the limit of every (row group, cell)
    uint64_t structure_epoch;  // calls so far that can move rows or re-map cells (rl_internal_structure_changed)
    cudaStream_t stream;
    int device;
};

// per-engine state owned by rl_maint.cu (freed through ext_free at rl_engine_destroy)
typedef int (*rl_ns_hook_fn)(rl_engine*, cudaStream_t, uint32_t n, const void* d_recs, int record_bytes,
                             const uint8_t* d_limited, const uint32_t* d_first_limited);

// Selects the engine's device, makes the caller's stream wait for every pipelined call, uploads pending limit tables
// and describes the table.  RL_OK or an error status (rl_last_error set).
int rl_internal_view(rl_engine* e, RlTableView* out);
int rl_internal_fail(rl_engine* e, int status, const char* msg);
void rl_internal_launched(rl_engine* e, uint32_t kernels);
uint32_t rl_internal_sm_count(rl_engine* e);  // streaming multiprocessors of the engine's device
void** rl_internal_ext(rl_engine* e, void (*ext_free)(void*));  // slot for rl_maint.cu's state (sets the deleter)
void rl_internal_set_ns_hook(rl_engine* e, rl_ns_hook_fn fn);
// forget the hot-row table (rows move when a region is rebuilt); enqueued on the engine's stream
int rl_internal_reset_hot_rows(rl_engine* e);
// a call that can move rows or re-map cells ran (limits set or deleted, counters deleted, compaction, import): the next
// rl_counters_drain is a full one
void rl_internal_structure_changed(rl_engine* e);
// present[l] = the counters of limit l exist, as rl_counters_export lists them (l < n; n >= limits_cap)
void rl_internal_present(rl_engine* e, uint8_t* present, uint32_t n);
// the unqualified limits l with flags[l] != 0 (l < n) have a counter again (as after add_counter): host registry only
void rl_internal_mark_present(rl_engine* e, const uint8_t* flags, uint32_t n);
