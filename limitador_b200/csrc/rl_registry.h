// rl_registry.h — the limit registry: which (row group, cell) each limit takes, the device tables built from that,
// and the rules that read it.  Plain C++ with no CUDA include, so that the engine (rl_engine.cu) and the host emulators
// (tests/emu) run this one copy.
#pragma once
#include <stdint.h>

#include <algorithm>
#include <cstring>
#include <map>
#include <string>
#include <utility>
#include <vector>

#include "../../include/rl_engine.h"
#include "rl_core.h"

struct HostLimit {
    bool defined = false;
    uint32_t ns = 0, varset = 0, qualified = 0;
    uint64_t max_value = 0, window_us = 0;
    uint32_t group = 0, cell = 0;
    bool simple_present = false;  // unqualified: entry exists in simple_limits (in_memory.rs:14)
};
struct HostGroup {
    uint32_t ns = 0, varset = 0, qualified = 0;
    uint32_t limit_of_cell[RL_MAX_CELLS];
    HostGroup() {
        for (auto& l : limit_of_cell) l = RL_NONE_U32;
    }
};

// What the calls need to know of the uploaded tables.
struct RlTableShape {
    uint32_t max_cells_used = 1;  // highest cell index + 1 over all row groups
    bool any_multi_ns = false;    // some namespace spans several rows
    uint32_t max_ns_limits = 0;   // the most limits of one namespace
    // remaining / ttl slots per record: the most limits of a namespace when some namespace spans several rows (the
    // records are then resolved into accesses, in the wide encoding past RL_MAX_CTRS_PER_REQ), else a row's cells
    uint32_t record_stride(uint32_t cells) const { return any_multi_ns ? std::max<uint32_t>(1, max_ns_limits) : cells; }
};

// The device tables as host arrays (RlDev: desc, limits, ns, ns_limit_ids; k_scan: group_ns).
struct RlTableImage {
    std::vector<RlCellDesc> desc;  // [groups][8]
    std::vector<RlLimitDev> lim;
    std::vector<RlNsDev> ns;
    std::vector<uint32_t> ns_ids, group_ns;
    RlTableShape shape;
};

struct RlRegistry {
    uint32_t cells = 1;  // cells per row
    std::vector<HostLimit> limits;
    std::vector<HostGroup> groups = std::vector<HostGroup>(1);  // [0] unused
    std::map<std::pair<uint32_t, uint32_t>, std::vector<uint32_t>> groups_by_key;
    std::vector<std::vector<uint32_t>> ns_limits;  // registration order
    bool dirty = true;                             // the tables changed since the last upload

    const HostLimit* find(uint32_t id) const { return id < limits.size() && limits[id].defined ? &limits[id] : nullptr; }

    // the limit's counters exist: qualified ones always, unqualified ones while simple_present (in_memory.rs:14,38-44)
    bool present(uint32_t id) const {
        const HostLimit* l = find(id);
        return l && (l->qualified || l->simple_present);
    }
    // an unqualified limit's simple_limits entry appears or goes (no effect on qualified or undefined limits)
    void set_simple_present(uint32_t id, bool on) {
        if (find(id) && !limits[id].qualified) limits[id].simple_present = on;
    }

    // f(id, limit) for every defined limit, in id order
    template <class F>
    void each(F&& f) const {
        for (size_t id = 0; id < limits.size(); id++)
            if (limits[id].defined) f((uint32_t)id, limits[id]);
    }

    // rl_limits_set: limits of one (namespace, variable set) share a row group with a free cell.  Stops at the first
    // refused limit, with the earlier ones applied; RL_OK, or RL_FATAL and *err.
    int set(const rl_limit_desc* limits_in, uint32_t n, std::string* err) {
        auto refuse = [&](std::string msg) {
            *err = std::move(msg);
            return RL_FATAL;
        };
        for (uint32_t i = 0; i < n; i++) {
            const rl_limit_desc& d = limits_in[i];
            if (d.limit_id == RL_NONE_U32) return refuse("limit_id 0xFFFFFFFF is reserved");
            if (d.limit_id > (1u << 26) || d.ns_id > (1u << 26))
                return refuse("limit_id / ns_id must be dense (<= 2^26)");
            const uint32_t q = d.qualified ? 1 : 0;
            const uint32_t varset = q ? d.varset_id : 0;
            if (q && d.varset_id == 0) return refuse("qualified limits need varset_id != 0");
            if (d.limit_id >= limits.size()) limits.resize(d.limit_id + 1);
            HostLimit& l = limits[d.limit_id];
            if (l.defined) {
                // Storage::update_limit (storage/mod.rs:67-83): identity fixed, max_value swapped
                if (l.ns != d.ns_id || l.window_us != d.window_us || l.qualified != q || l.varset != varset)
                    return refuse("limit " + std::to_string(d.limit_id) +
                                  ": namespace/window/variables are part of a limit's identity");
                if (l.max_value != d.max_value) {
                    l.max_value = d.max_value;
                    dirty = true;
                }
                if (!q) l.simple_present = true;  // add_counter: entry().or_default() (in_memory.rs:38-44)
                continue;
            }
            // pick a row group with a free cell
            auto& glist = groups_by_key[{d.ns_id, varset}];
            uint32_t g = 0, c = 0;
            for (uint32_t cand : glist) {
                for (uint32_t k = 0; k < cells; k++)
                    if (groups[cand].limit_of_cell[k] == RL_NONE_U32) {
                        g = cand;
                        c = k;
                        break;
                    }
                if (g) break;
            }
            if (!g) {
                if (groups.size() >= 0xFFFFFFF0u) return refuse("too many row groups");
                g = (uint32_t)groups.size();
                groups.emplace_back();
                groups[g].ns = d.ns_id;
                groups[g].varset = varset;
                groups[g].qualified = q;
                glist.push_back(g);
                c = 0;
            }
            groups[g].limit_of_cell[c] = d.limit_id;
            l.defined = true;
            l.ns = d.ns_id;
            l.varset = varset;
            l.qualified = q;
            l.max_value = d.max_value;
            l.window_us = d.window_us;
            l.group = g;
            l.cell = c;
            l.simple_present = !q;
            if (d.ns_id >= ns_limits.size()) ns_limits.resize(d.ns_id + 1);
            ns_limits[d.ns_id].push_back(d.limit_id);
            dirty = true;
        }
        return RL_OK;
    }

    // rl_limits_delete: the limits leave their cells and their namespaces (undefined ids are skipped)
    void remove(const uint32_t* ids, uint32_t n) {
        for (uint32_t i = 0; i < n; i++) {
            if (!find(ids[i])) continue;
            HostLimit& l = limits[ids[i]];
            groups[l.group].limit_of_cell[l.cell] = RL_NONE_U32;
            auto& v = ns_limits[l.ns];
            v.erase(std::remove(v.begin(), v.end(), ids[i]), v.end());
            l = HostLimit();
            dirty = true;
        }
    }

    // The device tables: cell descriptors per row group, limits, namespaces (single-row namespaces get mode 1 and
    // their packed cell list, the others mode 2).
    RlTableImage image() const {
        RlTableImage t;
        const size_t ngroups = groups.size();
        t.desc.assign(ngroups * 8, RlCellDesc{0, 0, RL_NONE_U32, 0});
        t.group_ns.assign(ngroups, 0);
        for (size_t g = 1; g < ngroups; g++) {
            t.group_ns[g] = groups[g].ns;
            for (uint32_t c = 0; c < RL_MAX_CELLS; c++) {
                const uint32_t lid = groups[g].limit_of_cell[c];
                if (lid == RL_NONE_U32) continue;
                t.shape.max_cells_used = std::max(t.shape.max_cells_used, c + 1);
                const HostLimit& l = limits[lid];
                t.desc[g * 8 + c] = RlCellDesc{l.max_value, l.window_us, lid, l.qualified};
            }
        }
        t.lim.assign(std::max<size_t>(limits.size(), 1), RlLimitDev{0, 0, 0, 0});
        each([&](uint32_t id, const HostLimit& l) { t.lim[id] = RlLimitDev{l.group, l.cell, l.ns, l.qualified}; });
        t.ns.resize(std::max<size_t>(ns_limits.size(), 1));
        for (size_t n = 0; n < t.ns.size(); n++) {
            RlNsDev& ns = t.ns[n];
            memset(&ns, 0, sizeof(RlNsDev));
            if (n >= ns_limits.size() || ns_limits[n].empty()) continue;
            const auto& L = ns_limits[n];
            ns.lim_off = (uint32_t)t.ns_ids.size();
            ns.lim_cnt = (uint32_t)L.size();
            t.shape.max_ns_limits = std::max<uint32_t>(t.shape.max_ns_limits, (uint32_t)L.size());
            bool single = L.size() <= RL_MAX_CELLS;
            for (uint32_t lid : L) {
                t.ns_ids.push_back(lid);
                if (limits[lid].group != limits[L[0]].group) single = false;
            }
            if (single) {
                ns.mode = 1;
                ns.group = limits[L[0]].group;
                ns.qualified_row = limits[L[0]].qualified;
                uint32_t cells_packed = 0;
                for (size_t k = 0; k < L.size(); k++) cells_packed |= limits[L[k]].cell << (4 * k);
                ns.cells = cells_packed | ((uint32_t)L.size() << 28);
            } else {
                ns.mode = 2;
                t.shape.any_multi_ns = true;
            }
        }
        if (t.ns_ids.empty()) t.ns_ids.push_back(0);
        return t;
    }
};
