// rl_match_records.h — the matcher's limits as records (library-internal; not part of include/).  What GET /limits and
// GET /counters (rl_rls.cpp) render a Limit from.
#pragma once
#include <stdint.h>

#include <string>
#include <vector>

struct rl_matcher;

struct RlLimitRecord {
    uint32_t limit_id = 0, varset_id = 0;
    uint64_t max_value = 0, seconds = 0;
    bool has_name = false;
    std::string name;
    std::vector<std::string> conditions, variables;  // the identity's sorted, unique sources (variables: the digest order)
};

// The live limits of namespace ns in counter order (the image's ns_lims order), taken under the matcher's shared lock.
// false: no limit was ever added for the namespace.
bool rl_matcher_ns_limit_records(rl_matcher* m, const std::string& ns, std::vector<RlLimitRecord>& out);
