// rl_match_records.h — the matcher's limits as records (library-internal; not part of include/).  What GET /limits and
// GET /counters (rl_rls.cpp) render a Limit from.
#pragma once
#include <stdint.h>

#include <functional>
#include <string>
#include <vector>

#include "rl_rls.h"

struct rl_matcher;

struct RlLimitRecord {
    uint32_t limit_id = 0, varset_id = 0;
    uint64_t max_value = 0, seconds = 0;
    bool has_name = false, has_id = false;
    std::string name, id;
    std::vector<std::string> conditions, variables;  // the identity's sorted, unique sources (variables: the digest order)
};

// The live limits of namespace ns in counter order (the image's ns_lims order), taken under the matcher's shared lock.
// false: no limit was ever added for the namespace.
bool rl_matcher_ns_limit_records(rl_matcher* m, const std::string& ns, std::vector<RlLimitRecord>& out);

// rl_matcher_configure's staged change (rl_rls_configure, include/rl_rls.h).  set[k] is a limit the engine must register
// (set_added[k] = 1) or whose max_value changed from old_max[k] (0), and came from entry set_entry[k]; deleted holds the
// live limits absent from the new set.
struct RlConfigurePlan {
    std::vector<rl_limit_desc> set;
    std::vector<uint32_t> set_entry;
    std::vector<uint8_t> set_added;
    std::vector<uint64_t> old_max;
    std::vector<uint32_t> deleted;
    uint32_t kept = 0, added = 0, updated = 0;
    uint32_t refused = 0xFFFFFFFFu;  // the entry the error names, if one does
    std::string error;
};

// Configure the matcher to hold exactly the limits of specs (Limitador's RateLimiter::configure_with), all or nothing, under
// the matcher's writer lock.  Every entry is parsed and the namespaces' sizes checked against min(max_limits_per_ns, the
// counter cap) before anything changes; the new tables are staged on a copy; apply(plan) runs on the staged plan (the
// caller's engine calls) and the copy replaces the tables only if it returns RL_OK.  dry_run: stage and count, no apply, no
// change.  RL_FATAL with plan.refused / plan.error for a refused entry; apply's status otherwise.
int rl_matcher_configure(rl_matcher* m, const rl_limit_spec* specs, uint32_t n, uint32_t max_limits_per_ns, bool dry_run,
                         RlConfigurePlan& plan, const std::function<int(RlConfigurePlan&)>& apply);
