// emu_cvars_snap.cpp — TEST-ONLY host driver of the dictionary's snapshot kernels (k_counter_vars_export, _check, _import
// in limitador_b200/csrc/rl_cvars_dev.cuh) under tests/emu/cuda_shim.h, or with -DEMU_SIMT under tests/emu/cuda_simt.h.
// It includes emu_cvars.cpp, so one library records (plan + k_counter_vars_record), exports and imports.  The call
// sequences follow rl_cv_dev_export / rl_cv_dev_import in rl_rls_dev.cu, with host loops in place of the CUB scans; the
// live counters rl_counters_export would list are the caller's.  Not shipped, not a fallback.  Also compiled into
// tests/san/san_cvars_snap.cpp for the ASan + UBSan run.
#include "emu_cvars.cpp"

#include <unordered_map>

namespace {

template <class T>
std::vector<unsigned long long> exclusive_sum(const T* x, uint64_t n) {
    std::vector<unsigned long long> out(n);
    unsigned long long acc = 0;
    for (uint64_t i = 0; i < n; i++) {
        out[i] = acc;
        acc += x[i];
    }
    return out;
}

// varset -> (first variable, variables) of the image's qualified limits, as rl_cv_dev_import builds it
std::vector<uint32_t> varset_table(const RlImage& I) {
    uint32_t n_vs = 1;
    for (uint32_t l = 0; l < I.n_limits; l++) n_vs = std::max(n_vs, I.lims[5ull * l + 4] + 1);
    std::vector<uint32_t> t(2ull * n_vs, 0);
    for (uint32_t l = 0; l < I.n_limits; l++) {
        const uint32_t* L = I.lims + 5ull * l;
        if (L[4] && L[3]) {
            t[2ull * L[4]] = L[2];
            t[2ull * L[4] + 1] = L[3];
        }
    }
    return t;
}

}  // namespace

extern "C" {

// The export of the entries the n live counters reference.  Returns the entries; *bytes = their blobs' bytes.  Writes
// only when cap and bytes_cap are large enough.
uint64_t emu_cvs_export(void* h, const uint32_t* image, uint64_t n, const uint32_t* lid, const uint64_t* lo, const uint64_t* hi,
                        uint64_t cap, uint64_t bytes_cap, uint32_t* varset, uint64_t* key_lo, uint64_t* key_hi, uint64_t* blob_off,
                        uint8_t* blobs, uint64_t* bytes) {
    EmuDict* d = static_cast<EmuDict*>(h);
    const uint64_t slots = d->slots.size();
    std::vector<uint8_t> mark(slots + 1, 0);
    std::vector<unsigned long long> len(slots + 1);
    CvMarkArgs a{lid, lo, hi, n, rl_img_view(image, image), d->view(), mark.data()};
    shim_launch(grid(n), kThreads, [&] { k_counter_vars_mark(a); });
    const CvDict D = d->view();
    shim_launch(grid(slots + 1), kThreads, [&] { k_counter_vars_kept(D, mark.data(), len.data()); });
    const std::vector<unsigned long long> pos = exclusive_sum(len.data(), slots + 1), idx = exclusive_sum(mark.data(), slots + 1);
    const uint64_t count = idx[slots];
    *bytes = pos[slots];
    if (cap == 0 || cap < count || bytes_cap < pos[slots]) return count;
    CvExportArgs e{D, mark.data(), pos.data(), idx.data(), varset, key_lo, key_hi, blob_off, blobs};
    shim_launch(grid(slots + 1), kThreads, [&] { k_counter_vars_export(e); });
    return count;
}

// The import: 0 (RL_OK), RL_FATAL with *bad = entry << 8 | reason, or RL_TRANSIENT (*bad = 0 for the arena, 1 for a slot).
int emu_cvs_import(void* h, const uint32_t* image, uint64_t n, const uint32_t* varset, const uint64_t* key_lo, const uint64_t* key_hi,
                   const uint64_t* blob_off, const uint8_t* blobs, uint64_t* added, uint64_t* bad) {
    EmuDict* d = static_cast<EmuDict*>(h);
    *added = 0;
    *bad = RL_CV_GOOD;
    if (n == 0) return RL_OK;
    for (uint64_t i = 0; i < n; i++)
        if (blob_off[i + 1] < blob_off[i]) {
            *bad = i << 8;
            return RL_FATAL;
        }
    const RlImage img = rl_img_view(image, image);
    const std::vector<uint32_t> vt = varset_table(img);
    std::vector<unsigned long long> len(n + 1), word(1, RL_CV_GOOD);
    CvImportArgs a{varset, key_lo, key_hi, blob_off, blobs, n, img, vt.data(), (uint32_t)(vt.size() / 2), d->view(), len.data(),
                   nullptr, 0, word.data()};
    shim_launch(grid(n + 1), kThreads, [&] { k_counter_vars_check(a); });
    const std::vector<unsigned long long> pos = exclusive_sum(len.data(), n + 1);
    a.pos = pos.data();
    const uint64_t slots = d->slots.size();
    std::vector<uint8_t> mark(slots + 1, 0);
    std::vector<unsigned long long> klen(slots + 1);
    const CvDict D = d->view();
    shim_launch(grid(slots), kThreads, [&] { k_counter_vars_occupied(D, mark.data()); });
    shim_launch(grid(slots + 1), kThreads, [&] { k_counter_vars_kept(D, mark.data(), klen.data()); });
    const std::vector<unsigned long long> kpos = exclusive_sum(klen.data(), slots + 1);
    if (word[0] != RL_CV_GOOD) {
        *bad = word[0];
        return RL_FATAL;
    }
    if (pos[n] == 0) return RL_OK;  // every key is held already
    if (pos[n] + kpos[slots] > d->arena.size()) {
        *bad = 0;
        return RL_TRANSIENT;
    }
    EmuDict to;
    to.slots.assign(slots, CvSlot{});
    to.arena.assign(d->arena.size(), 0);
    to.ctl.assign(RL_CV_CTL_WORDS, 0);
    to.ctl[RL_CV_DROPPED] = d->ctl[RL_CV_DROPPED];
    CvRebuildArgs b{D, mark.data(), kpos.data(), to.view()};
    shim_launch(grid(slots + 1), kThreads, [&] { k_counter_vars_rebuild(b); });
    a.dict = to.view();
    a.base = kpos[slots];
    // the import's claims race in 256-thread blocks under the fiber emulator, as the recording's do
    shim_launch((uint32_t)((n + 1 + kRecordThreads - 1) / kRecordThreads), kRecordThreads, [&] { k_counter_vars_import(a); });
    if (word[0] != RL_CV_GOOD) {  // as rl_cv_dev_import: name the later entry of the first repeated key
        std::unordered_map<uint64_t, uint64_t> seen;
        for (uint64_t i = 0; i < n; i++) {
            const uint64_t f = rl_cv_fp(varset[i], key_lo[i], key_hi[i]);
            auto it = seen.find(f);
            if (it != seen.end() && varset[it->second] == varset[i] && key_lo[it->second] == key_lo[i] && key_hi[it->second] == key_hi[i]) {
                *bad = i << 8 | RL_CV_BAD_DUPLICATE;
                return RL_FATAL;
            }
            seen.emplace(f, i);
        }
        *bad = word[0];
        return RL_FATAL;
    }
    if (to.ctl[RL_CV_DROPPED] != d->ctl[RL_CV_DROPPED]) {
        *bad = 1;
        return RL_TRANSIENT;
    }
    *added = to.ctl[RL_CV_KEYS] - d->ctl[RL_CV_KEYS];
    std::swap(d->slots, to.slots);
    std::swap(d->arena, to.arena);
    std::swap(d->ctl, to.ctl);
    return RL_OK;
}

// rl_cv_check_entry on one blob (for the sanitizer fuzz and the Python tests of single entries)
uint32_t emu_cvs_check_entry(const uint32_t* image, uint32_t vs, uint64_t lo, uint64_t hi, const uint8_t* b, uint64_t n) {
    const RlImage img = rl_img_view(image, image);
    const std::vector<uint32_t> vt = varset_table(img);
    return rl_cv_check_entry(img, vt.data(), (uint32_t)(vt.size() / 2), vs, lo, hi, b, n);
}

}  // extern "C"
