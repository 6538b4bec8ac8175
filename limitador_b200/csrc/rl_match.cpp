// rl_match.cpp — CPU front: limits -> counters (include/rl_match.h, SURVEY.md §8 f1).
//
// Host-only code.  The reference walks a CEL AST per condition and per variable for every limit of the
// namespace (limit.rs:157-174, cel.rs:185-227,314-334), building string maps on the way; here every
// operand of every accepted expression is interned into a SLOT when the limit is added, a request's
// bindings are dropped into the slot array once, and a limit is a list of TESTS plus a list of slots that
// must be present.  A test is a presence test on one slot, or up to RL_MATCH_MAX_ATOMS value atoms over one
// slot and the truth table of the boolean formula that combines them (`x == 'a'` is one atom and the table
// 0b10, `x != 'a'` the table 0b01).  The counter key of a variable set is digested once per request and
// shared by the limits that use the same variables.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <shared_mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "rl_blake2b.h"
#include "rl_error.h"
#include "rl_match.h"
#include "rl_match_image.h"
#include "rl_match_records.h"

namespace {

using rl_b2::KeyDigest;  // rl_blake2b.h: the same digest as the device plan

// ---- operand slots ------------------------------------------------------------------------
struct SlotKey {
    uint32_t desc;
    std::string key;
};

struct SlotTable {
    std::vector<int32_t> idx;  // open addressing, -1 = empty
    std::vector<SlotKey> keys;
    SlotTable() : idx(64, -1) {}
    static uint64_t hash(uint32_t desc, const char* k, size_t n) {
        uint64_t h = 0xcbf29ce484222325ULL ^ desc;
        h *= 0x100000001b3ULL;
        for (size_t i = 0; i < n; i++) {
            h ^= (uint8_t)k[i];
            h *= 0x100000001b3ULL;
        }
        return h ^ (h >> 29);
    }
    int find(uint32_t desc, const char* k, size_t n) const {
        const uint64_t mask = idx.size() - 1;
        for (uint64_t p = hash(desc, k, n) & mask;; p = (p + 1) & mask) {
            const int32_t s = idx[p];
            if (s < 0) return -1;
            const SlotKey& sk = keys[s];
            if (sk.desc == desc && sk.key.size() == n && memcmp(sk.key.data(), k, n) == 0) return s;
        }
    }
    uint32_t intern(uint32_t desc, const std::string& k) {
        const int f = find(desc, k.data(), k.size());
        if (f >= 0) return (uint32_t)f;
        keys.push_back({desc, k});
        if (keys.size() * 2 > idx.size()) {
            idx.assign(idx.size() * 2, -1);
            for (size_t s = 0; s + 1 < keys.size(); s++) place((int32_t)s);
        }
        place((int32_t)keys.size() - 1);
        return (uint32_t)keys.size() - 1;
    }
    void place(int32_t s) {
        const uint64_t mask = idx.size() - 1;
        uint64_t p = hash(keys[s].desc, keys[s].key.data(), keys[s].key.size()) & mask;
        while (idx[p] >= 0) p = (p + 1) & mask;
        idx[p] = s;
    }
};

// a value atom: RL_ATOM_* against one literal, or against a list of them for RL_ATOM_IN
struct Atom {
    uint32_t op;
    std::vector<std::string> lits;
};

// a test of one operand (see rl_match_image.h): no atoms = present; else table bit `atom bits` of its value
struct Test {
    uint32_t slot;
    std::vector<Atom> atoms;
    uint64_t table;
};

// a test as parsed, before its operand is interned
struct ParsedTest {
    uint32_t desc;
    std::string key;
    std::vector<Atom> atoms;
    uint64_t table;
};

struct MLimit {
    std::string ns, name, id;
    bool has_name = false, has_id = false, deleted = false;
    uint32_t ns_id = 0, varset_id = 0;
    uint64_t max_value = 0, seconds = 0;
    std::vector<std::string> conds, vars;  // sorted, unique (the identity)
    std::vector<Test> tests;
    std::vector<uint32_t> var_slots;  // same order as vars
};

// ---- the accepted expression grammar (see rl_match.h) -----------------------------------------
inline bool is_ident_start(unsigned char c) { return c == '_' || (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z'); }
inline bool is_word(unsigned char c) { return is_ident_start(c) || (c >= '0' && c <= '9'); }  // CEL identifiers are ASCII
inline void skip_ws(const char*& p) {
    while (*p == ' ' || *p == '\t' || *p == '\n' || *p == '\r' || *p == '\f' || *p == '\v') p++;
}

bool parse_operand(const char*& p, uint32_t& desc, std::string& key) {
    skip_ws(p);
    static const char kDesc[] = "descriptors[";
    if (strncmp(p, kDesc, sizeof kDesc - 1) == 0 && p[sizeof kDesc - 1] >= '0' && p[sizeof kDesc - 1] <= '9') {
        const char* q = p + sizeof kDesc - 1;
        uint64_t n = 0;
        while (*q >= '0' && *q <= '9') {
            n = n * 10 + (uint64_t)(*q - '0');
            if (n >= RL_BIND_ROOT) return false;
            q++;
        }
        if (*q != ']') return false;
        q++;
        if (*q == '.') {
            q++;
            if (!is_ident_start((unsigned char)*q)) return false;
            const char* s = q;
            while (is_word((unsigned char)*q)) q++;
            key.assign(s, q);
        } else if (*q == '[') {
            q++;
            const char kq = *q;
            if (kq != '\'' && kq != '"') return false;
            q++;
            const char* s = q;
            // the closing quote must be the opening one (CEL rejects descriptors[0]['k"] at parse time) and the
            // key must not need CEL's escape processing, which this subset does not do: refuse instead
            while (*q && *q != kq && *q != '\\') q++;
            if (*q != kq || q == s) return false;
            key.assign(s, q);
            q++;
            if (*q != ']') return false;
            q++;
        } else {
            return false;
        }
        desc = (uint32_t)n;
        p = q;
        return true;
    }
    if (!is_ident_start((unsigned char)*p)) return false;
    const char* s = p;
    while (is_word((unsigned char)*p)) p++;
    // `req.method` is member access on the variable `req` in CEL, not a root binding named "req.method"
    // (the reference would never apply such a limit: Predicate::test fails on the unbound `req`,
    // limit/cel.rs:314-322); dotted keys are only reachable as descriptors[0]['req.method'].  Refused.
    if (*p == '.') return false;
    key.assign(s, p);
    desc = RL_BIND_ROOT;
    return true;
}

bool parse_condition(const char* src, uint32_t& desc, std::string& key, bool& neq, std::string& lit) {
    const char* p = src;
    if (!parse_operand(p, desc, key)) return false;
    skip_ws(p);
    if (p[0] == '=' && p[1] == '=') neq = false;
    else if (p[0] == '!' && p[1] == '=') neq = true;
    else return false;
    p += 2;
    skip_ws(p);
    const char quote = *p;
    if (quote != '\'' && quote != '"') return false;
    p++;
    const char* s = p;
    // a literal that needs CEL's escape processing ("a\nb") would compare differently here: refused
    while (*p && *p != quote && *p != '\\') p++;
    if (*p != quote) return false;
    lit.assign(s, p);
    p++;
    skip_ws(p);
    return *p == 0;
}

bool parse_variable(const char* src, uint32_t& desc, std::string& key) {
    const char* p = src;
    if (!parse_operand(p, desc, key)) return false;
    skip_ws(p);
    return *p == 0;
}

// ---- the boolean dialect (RL_MATCH_DIALECT_BOOLEAN, see rl_match.h) ------------------------------
// A recursive-descent parser over a token list, then the normal form: the top-level && split into conjuncts, each one
// a presence test or an operand group (one operand, at most RL_MATCH_MAX_ATOMS atoms) compiled to its truth table.
// Everything the normal form does not hold is refused on the parsed form.
class BoolParser {
  public:
    explicit BoolParser(const char* src) : src_(src) {}

    bool parse(std::vector<ParsedTest>& out) {
        if (!lex()) return false;
        int root;
        if (!parse_or(0, root) || tok_[pos_].kind != T_END) return false;
        std::vector<int> conj;
        split_and(root, conj);
        for (const int c : conj) {
            ParsedTest t;
            if (nodes_[c].kind == N_PRESENT) {  // only ever a top-level conjunct, and only positively
                t.desc = nodes_[c].desc;
                t.key = nodes_[c].key;
                t.table = 0;
                out.push_back(std::move(t));
                continue;
            }
            std::vector<int> atoms;
            if (!group_atoms(c, atoms) || atoms.size() > RL_MATCH_MAX_ATOMS) return false;
            t.desc = nodes_[atoms[0]].desc;
            t.key = nodes_[atoms[0]].key;
            for (const int a : atoms) {
                if (nodes_[a].desc != t.desc || nodes_[a].key != t.key) return false;  // || or ! spanning two operands
                t.atoms.push_back(nodes_[a].atom);
            }
            t.table = 0;
            for (uint32_t bits = 0; bits < (1u << atoms.size()); bits++)
                if (eval(c, atoms, bits)) t.table |= 1ull << bits;
            out.push_back(std::move(t));
        }
        return true;
    }

  private:
    enum TokKind { T_END, T_IDENT, T_STR, T_INT, T_PUNCT };
    struct Tok {
        TokKind kind;
        std::string text;  // identifier, unquoted string, digits or punctuation
    };
    enum NodeKind { N_ATOM, N_PRESENT, N_NOT, N_AND, N_OR };
    struct Node {
        NodeKind kind;
        int a = -1, b = -1;  // operands of N_NOT (a), N_AND / N_OR (a, b)
        uint32_t desc = 0;   // N_ATOM / N_PRESENT: the operand
        std::string key;
        Atom atom;           // N_ATOM
        bool negated = false;  // N_ATOM: written with !=
        bool relation = false;  // an ==, != or `in` not inside parentheses
    };
    static constexpr int kMaxDepth = 32;  // nesting of ( and !

    const char* src_;
    std::vector<Tok> tok_;
    size_t pos_ = 0;
    std::vector<Node> nodes_;

    bool lex() {
        const char* p = src_;
        for (;;) {
            skip_ws(p);
            if (!*p) break;
            const unsigned char c = (unsigned char)*p;
            if (is_ident_start(c)) {
                const char* s = p;
                while (is_word((unsigned char)*p)) p++;
                if (*p == '\'' || *p == '"') return false;  // r'..', b'..': raw and byte strings
                tok_.push_back({T_IDENT, std::string(s, p)});
            } else if (c >= '0' && c <= '9') {
                const char* s = p;
                while (*p >= '0' && *p <= '9') p++;
                tok_.push_back({T_INT, std::string(s, p)});
            } else if (c == '\'' || c == '"') {
                if (p[1] == *p && p[2] == *p) return false;  // triple-quoted
                const char q = *p++;
                const char* s = p;
                // no escape processing here: a backslash anywhere refuses the expression, as in the table dialect
                while (*p && *p != q && *p != '\\' && *p != '\n' && *p != '\r') p++;
                if (*p != q) return false;
                tok_.push_back({T_STR, std::string(s, p)});
                p++;
            } else {
                static const char* const kPunct[] = {"&&", "||", "==", "!=", "(", ")", "[", "]", ".", ",", "!"};
                bool hit = false;
                for (const char* k : kPunct) {
                    const size_t n = strlen(k);
                    if (strncmp(p, k, n) == 0) {
                        tok_.push_back({T_PUNCT, k});
                        p += n;
                        hit = true;
                        break;
                    }
                }
                if (!hit) return false;
            }
        }
        tok_.push_back({T_END, ""});
        return true;
    }

    bool is(TokKind k, const char* text = nullptr, size_t ahead = 0) const {
        const size_t i = std::min(pos_ + ahead, tok_.size() - 1);
        return tok_[i].kind == k && (!text || tok_[i].text == text);
    }
    bool take(TokKind k, const char* text = nullptr) {
        if (!is(k, text)) return false;
        pos_++;
        return true;
    }
    int node(Node n) {
        nodes_.push_back(std::move(n));
        return (int)nodes_.size() - 1;
    }

    static bool reserved(const std::string& w) {
        static const char* const kWords[] = {"true",  "false",    "null",     "in",     "as",     "break",   "const",
                                             "continue", "else",  "for",      "function", "if",   "import",  "let",
                                             "loop",  "package",  "namespace", "return", "var",   "void",    "while",
                                             "descriptors", "has"};
        for (const char* k : kWords)
            if (w == k) return true;
        return false;
    }

    // descriptors[N] after the identifier: N into desc
    bool descriptor_index(uint32_t& desc) {
        if (!take(T_PUNCT, "[") || !is(T_INT)) return false;
        uint64_t n = 0;
        for (const char d : tok_[pos_].text) {
            n = n * 10 + (uint64_t)(d - '0');
            if (n >= RL_BIND_ROOT) return false;
        }
        pos_++;
        desc = (uint32_t)n;
        return take(T_PUNCT, "]");
    }

    // IDENT | descriptors[N].IDENT | descriptors[N]['key']
    bool operand(uint32_t& desc, std::string& key) {
        if (!is(T_IDENT)) return false;
        if (tok_[pos_].text != "descriptors") {
            if (reserved(tok_[pos_].text)) return false;
            key = tok_[pos_++].text;
            desc = RL_BIND_ROOT;
            return true;
        }
        pos_++;
        if (!descriptor_index(desc)) return false;
        if (take(T_PUNCT, ".")) {
            if (!is(T_IDENT)) return false;
            key = tok_[pos_++].text;
            return true;
        }
        if (!take(T_PUNCT, "[") || !is(T_STR) || tok_[pos_].text.empty()) return false;
        key = tok_[pos_++].text;
        return take(T_PUNCT, "]");
    }

    bool parse_or(int depth, int& out) {
        if (!parse_and(depth, out)) return false;
        while (take(T_PUNCT, "||")) {
            int r;
            if (!parse_and(depth, r)) return false;
            Node n{N_OR};
            n.a = out;
            n.b = r;
            out = node(std::move(n));
        }
        return true;
    }

    bool parse_and(int depth, int& out) {
        if (!parse_unary(depth, out)) return false;
        while (take(T_PUNCT, "&&")) {
            int r;
            if (!parse_unary(depth, r)) return false;
            Node n{N_AND};
            n.a = out;
            n.b = r;
            out = node(std::move(n));
        }
        return true;
    }

    // an ==, != or `in` binds looser than a leading `!` in CEL (`!x == 'a'` is `(!x) == 'a'` there): refused after a `!`
    bool parse_unary(int depth, int& out) {
        if (depth > kMaxDepth) return false;
        if (take(T_PUNCT, "!")) {
            int a;
            if (!(is(T_PUNCT, "!") || is(T_PUNCT, "(") || is(T_IDENT)) || !parse_unary(depth + 1, a)) return false;
            if (nodes_[a].relation) return false;
            Node n{N_NOT};
            n.a = a;
            out = node(std::move(n));
            return true;
        }
        return parse_primary(depth, out);
    }

    bool parse_primary(int depth, int& out) {
        if (take(T_PUNCT, "(")) {
            if (!parse_or(depth + 1, out) || !take(T_PUNCT, ")")) return false;
            nodes_[out].relation = false;
            return true;
        }
        if (is(T_IDENT, "has") && is(T_PUNCT, "(", 1)) {  // has(descriptors[N].IDENT)
            pos_ += 2;
            Node n{N_PRESENT};
            if (!take(T_IDENT, "descriptors") || !descriptor_index(n.desc) || !take(T_PUNCT, ".") || !is(T_IDENT)) return false;
            n.key = tok_[pos_++].text;
            if (!take(T_PUNCT, ")")) return false;
            out = node(std::move(n));
            return true;
        }
        Node n{N_ATOM};
        if (is(T_STR)) {  // 'key' in descriptors[N], or 'lit' ==|!= operand
            const std::string lit = tok_[pos_++].text;
            if (take(T_IDENT, "in")) {
                Node p{N_PRESENT};
                if (lit.empty() || !take(T_IDENT, "descriptors") || !descriptor_index(p.desc)) return false;
                p.key = lit;
                p.relation = true;
                out = node(std::move(p));
                return true;
            }
            if (is(T_PUNCT, "==") || is(T_PUNCT, "!=")) {
                n.negated = tok_[pos_++].text == "!=";
                if (!operand(n.desc, n.key)) return false;
                n.atom = {RL_ATOM_EQ, {lit}};
                n.relation = true;
                out = node(std::move(n));
                return true;
            }
            return false;
        }
        if (!operand(n.desc, n.key)) return false;
        if (is(T_PUNCT, "==") || is(T_PUNCT, "!=")) {  // operand ==|!= 'lit'
            n.negated = tok_[pos_++].text == "!=";
            if (!is(T_STR)) return false;
            n.atom = {RL_ATOM_EQ, {tok_[pos_++].text}};
            n.relation = true;
            out = node(std::move(n));
            return true;
        }
        if (take(T_PUNCT, ".")) {  // operand.startsWith|endsWith|contains('lit')
            if (!is(T_IDENT)) return false;
            const std::string& f = tok_[pos_++].text;
            if (f == "startsWith") n.atom.op = RL_ATOM_PREFIX;
            else if (f == "endsWith") n.atom.op = RL_ATOM_SUFFIX;
            else if (f == "contains") n.atom.op = RL_ATOM_CONTAINS;
            else return false;
            if (!take(T_PUNCT, "(") || !is(T_STR)) return false;
            n.atom.lits.push_back(tok_[pos_++].text);
            if (!take(T_PUNCT, ")")) return false;
            out = node(std::move(n));
            return true;
        }
        if (take(T_IDENT, "in")) {  // operand in ['lit', ...] (possibly empty, no trailing comma)
            if (!take(T_PUNCT, "[")) return false;
            n.atom.op = RL_ATOM_IN;
            if (!take(T_PUNCT, "]")) {
                do {
                    if (!is(T_STR)) return false;
                    n.atom.lits.push_back(tok_[pos_++].text);
                } while (take(T_PUNCT, ","));
                if (!take(T_PUNCT, "]")) return false;
            }
            n.relation = true;
            out = node(std::move(n));
            return true;
        }
        return false;
    }

    void split_and(int n, std::vector<int>& out) const {
        if (nodes_[n].kind == N_AND) {
            split_and(nodes_[n].a, out);
            split_and(nodes_[n].b, out);
        } else {
            out.push_back(n);
        }
    }

    // the atoms of an operand group, left to right; false if a presence test sits inside it
    bool group_atoms(int n, std::vector<int>& out) const {
        const Node& x = nodes_[n];
        if (x.kind == N_PRESENT) return false;  // negated, or inside ||: refused
        if (x.kind == N_ATOM) {
            out.push_back(n);
            return true;
        }
        if (!group_atoms(x.a, out)) return false;
        return x.b < 0 || group_atoms(x.b, out);
    }

    // the group's formula with atom atoms[j] = bit j of `bits`
    bool eval(int n, const std::vector<int>& atoms, uint32_t bits) const {
        const Node& x = nodes_[n];
        switch (x.kind) {
            case N_ATOM: {
                const size_t j = (size_t)(std::find(atoms.begin(), atoms.end(), n) - atoms.begin());
                return (((bits >> j) & 1u) != 0) != x.negated;
            }
            case N_NOT: return !eval(x.a, atoms, bits);
            case N_AND: return eval(x.a, atoms, bits) && eval(x.b, atoms, bits);
            case N_OR: return eval(x.a, atoms, bits) || eval(x.b, atoms, bits);
            default: return false;
        }
    }
};

// a condition of the table dialect as a one-atom test
bool parse_table_condition(const char* src, ParsedTest& t) {
    bool neq;
    std::string lit;
    if (!parse_condition(src, t.desc, t.key, neq, lit)) return false;
    t.atoms = {Atom{RL_ATOM_EQ, {lit}}};
    t.table = neq ? 0x1 : 0x2;  // bit 1: the value equals the literal
    return true;
}

// per-thread request scratch: slot -> value of the current request (stamped, never cleared)
struct Scratch {
    std::vector<const char*> val;
    std::vector<uint64_t> stamp;
    uint64_t epoch = 0;
    struct VK {
        uint32_t varset;
        uint64_t lo, hi;
    };
    std::vector<VK> keys;
};
thread_local Scratch tls_scratch;

}  // namespace

struct MLock {
    std::shared_mutex mu;
    uint32_t counter_cap = RL_MAX_COUNTERS_PER_REQUEST;  // rl_matcher_set_counter_cap
    uint32_t dialect = RL_MATCH_DIALECT_TABLE;           // rl_matcher_set_dialect: how later add_limit calls parse
    std::mutex err_mu;  // last_error is also written by matching calls, which hold `mu` shared
    std::string last_error;
};

// Everything the limits define: rl_matcher_configure stages a whole new set of limits on a copy and swaps it in.
struct MTables {
    SlotTable slots;
    std::vector<MLimit> limits;
    std::unordered_map<std::string, uint32_t> ns_ids;
    std::vector<std::vector<uint32_t>> ns_limits;  // registration order
    std::map<std::string, uint32_t> by_identity;
    std::map<std::string, uint32_t> varsets;  // (namespace, variables) -> id, from 1
};

// The lock first and the tables behind it, in that order: matching threads bump the lock's reader count on every batch,
// and the tables they read stay off its cache line.
struct rl_matcher : MLock, MTables {
    uint64_t generation = 1;                  // rl_matcher_generation: bumped by every change of the limits or the cap
};

namespace {

template <class... A>
int mfail(rl_matcher* m, const char* fmt, A... a) {
    std::string msg = rl_format(fmt, a...);
    std::lock_guard<std::mutex> g(m->err_mu);
    m->last_error = std::move(msg);
    return RL_FATAL;
}

std::string joined(const std::vector<std::string>& v) {
    std::string s;
    for (const auto& x : v) {
        s += x;
        s.push_back('\x01');
    }
    return s;
}

// counters_that_apply for one request; returns RL_OK or RL_FATAL (capacity)
int match_one(const rl_matcher* m, uint32_t ns_id, const rl_binding* binds, uint32_t nb, rl_counter* out, uint64_t cap,
              uint64_t& n_out, Scratch& s) {
    n_out = 0;
    if (ns_id >= m->ns_limits.size()) return RL_OK;  // unknown namespace: no limits apply (lib.rs:434-440)
    const size_t nslots = m->slots.keys.size();
    if (s.val.size() < nslots) {
        s.val.resize(nslots, nullptr);
        s.stamp.resize(nslots, 0);
    }
    const uint64_t ep = ++s.epoch;
    for (uint32_t i = 0; i < nb; i++) {
        const rl_binding& b = binds[i];
        if (!b.key || !b.value) continue;
        const int slot = m->slots.find(b.descriptor, b.key, strlen(b.key));
        if (slot < 0) continue;  // nothing refers to this binding
        s.val[slot] = b.value;   // a HashMap holds one value per key: the last one given wins
        s.stamp[slot] = ep;
    }
    s.keys.clear();
    for (const uint32_t lid : m->ns_limits[ns_id]) {
        const MLimit& L = m->limits[lid];
        if (L.deleted) continue;
        bool ok = true;
        for (const Test& t : L.tests) {
            const char* v = (s.stamp[t.slot] == ep) ? s.val[t.slot] : nullptr;
            if (!v) {  // unbound name / missing key: the predicate is false (cel.rs:315-331)
                ok = false;
                break;
            }
            if (t.atoms.empty()) continue;  // a presence test: bound is all it asks
            const uint32_t n = (uint32_t)strlen(v);
            uint32_t bits = 0;
            for (size_t j = 0; j < t.atoms.size(); j++) {
                const Atom& a = t.atoms[j];
                bool hit = false;
                for (size_t k = 0; k < a.lits.size() && !hit; k++)
                    hit = rl_str_op(a.op == RL_ATOM_IN ? RL_ATOM_EQ : a.op, (const uint8_t*)v, n, (const uint8_t*)a.lits[k].data(),
                                    (uint32_t)a.lits[k].size());
                bits |= (uint32_t)hit << j;
            }
            if (!((t.table >> bits) & 1)) {
                ok = false;
                break;
            }
        }
        if (!ok) continue;
        for (const uint32_t vs : L.var_slots)
            if (s.stamp[vs] != ep) {  // a variable without a value: no counter (limit.rs:133-148, lib.rs:515-519)
                ok = false;
                break;
            }
        if (!ok) continue;
        // the engine takes at most RL_MAX_COUNTERS_PER_REQUEST counters per request: refuse here, before
        // anything is enqueued, instead of letting the device resolve fail the batch half-applied
        if (n_out >= cap || n_out >= m->counter_cap) return RL_FATAL;
        rl_counter& c = out[n_out++];
        c.limit_id = lid;
        c._pad = 0;
        c.key_lo = c.key_hi = 0;
        if (!L.var_slots.empty()) {
            bool hit = false;
            for (const auto& k : s.keys)
                if (k.varset == L.varset_id) {
                    c.key_lo = k.lo;
                    c.key_hi = k.hi;
                    hit = true;
                    break;
                }
            if (!hit) {
                KeyDigest d;
                for (size_t j = 0; j < L.vars.size(); j++) {
                    d.str(L.vars[j].data(), L.vars[j].size());
                    const char* v = s.val[L.var_slots[j]];
                    d.str(v, strlen(v));
                }
                d.finish(c.key_lo, c.key_hi);
                s.keys.push_back({L.varset_id, c.key_lo, c.key_hi});
            }
        }
    }
    return RL_OK;
}

// The identity (limit.rs:177-214) as by_identity keys it: namespace, seconds, the sorted condition and variable sets.
std::string identity_of(const MLimit& L) {
    return L.ns + '\0' + std::to_string(L.seconds) + '\0' + joined(L.conds) + '\0' + joined(L.vars);
}

// A limit as parsed (Limit::new), before any table of the matcher is touched.
struct ParsedLimit {
    MLimit L;
    std::vector<ParsedTest> conds;
    std::vector<std::pair<uint32_t, std::string>> vars;  // (descriptor, key) of each variable, in L.vars order
    std::string ident;                                   // the identity (limit.rs:177-214)
};

// The parse-only half of rl_matcher_add_limit_ex: false, with the reason in err, for an expression the dialect refuses.
bool parse_limit(uint32_t dialect, const char* ns, uint64_t max_value, uint64_t seconds, const char* const* conditions,
                 uint32_t n_cond, const char* const* variables, uint32_t n_var, const char* name, const char* id,
                 ParsedLimit& P, std::string& err) {
    MLimit& L = P.L;
    L.ns = ns;
    L.max_value = max_value;
    L.seconds = seconds;
    if (name) {
        L.name = name;
        L.has_name = true;
    }
    if (id) {
        L.id = id;
        L.has_id = true;
    }
    for (uint32_t i = 0; i < n_cond; i++) L.conds.emplace_back(conditions[i] ? conditions[i] : "");
    for (uint32_t i = 0; i < n_var; i++) L.vars.emplace_back(variables[i] ? variables[i] : "");
    // the identity holds SETS of expression sources (limit.rs:31-48: BTreeSet)
    std::sort(L.conds.begin(), L.conds.end());
    L.conds.erase(std::unique(L.conds.begin(), L.conds.end()), L.conds.end());
    std::sort(L.vars.begin(), L.vars.end());
    L.vars.erase(std::unique(L.vars.begin(), L.vars.end()), L.vars.end());
    for (size_t i = 0; i < L.conds.size(); i++) {
        bool ok;
        if (dialect == RL_MATCH_DIALECT_BOOLEAN) {
            ok = BoolParser(L.conds[i].c_str()).parse(P.conds);
        } else {
            P.conds.emplace_back();
            ok = parse_table_condition(L.conds[i].c_str(), P.conds.back());
        }
        if (!ok) {
            err = rl_format("unsupported condition expression: %s", L.conds[i].c_str());
            return false;
        }
    }
    P.vars.resize(L.vars.size());
    for (size_t i = 0; i < L.vars.size(); i++)
        if (!parse_variable(L.vars[i].c_str(), P.vars[i].first, P.vars[i].second)) {
            err = rl_format("unsupported variable expression: %s", L.vars[i].c_str());
            return false;
        }
    P.ident = identity_of(L);
    return true;
}

// The table half of rl_matcher_add_limit_ex (Storage::add_limit / update_limit) on t; returns the limit's id.
uint32_t place_limit(MTables& t, ParsedLimit&& P, int keep_existing, int* out_existed) {
    MLimit& L = P.L;
    uint32_t lid;
    auto it = t.by_identity.find(P.ident);
    if (it != t.by_identity.end()) {
        // update_limit (storage/mod.rs:67-83): same identity, new max_value / name; a deleted one comes back
        lid = it->second;
        MLimit& E = t.limits[lid];
        if (out_existed) *out_existed = E.deleted ? 0 : 1;
        // Storage::add_limit is a HashSet::insert: on an equal (live) element it is a no-op and the OLD
        // max_value / name stay (storage/mod.rs:60-65); only update_limit swaps them (:67-83)
        if (!(keep_existing && !E.deleted)) {
            // update_limit replaces the whole Limit, id included, only when max_value or name differ
            if (E.deleted || E.max_value != L.max_value || E.has_name != L.has_name || E.name != L.name) {
                E.id = L.id;
                E.has_id = L.has_id;
            }
            E.max_value = L.max_value;
            E.name = L.name;
            E.has_name = L.has_name;
        }
        if (E.deleted) {  // deleted and added again: it is the namespace's newest limit
            auto& order = t.ns_limits[E.ns_id];
            order.erase(std::remove(order.begin(), order.end(), lid), order.end());
            order.push_back(lid);
            E.deleted = false;
        }
        return lid;
    }
    lid = (uint32_t)t.limits.size();
    auto nit = t.ns_ids.find(L.ns);
    if (nit == t.ns_ids.end()) {
        nit = t.ns_ids.emplace(L.ns, (uint32_t)t.ns_ids.size()).first;
        t.ns_limits.emplace_back();
    }
    L.ns_id = nit->second;
    if (!L.vars.empty()) {
        const std::string vk = L.ns + '\0' + joined(L.vars);
        auto vit = t.varsets.find(vk);
        if (vit == t.varsets.end()) vit = t.varsets.emplace(vk, (uint32_t)t.varsets.size() + 1).first;
        L.varset_id = vit->second;
    }
    for (auto& c : P.conds) L.tests.push_back({t.slots.intern(c.desc, c.key), std::move(c.atoms), c.table});
    for (const auto& v : P.vars) L.var_slots.push_back(t.slots.intern(v.first, v.second));
    t.by_identity.emplace(std::move(P.ident), lid);
    t.ns_limits[L.ns_id].push_back(lid);
    t.limits.push_back(std::move(L));
    return lid;
}

rl_limit_desc desc_of(const MTables& t, uint32_t lid) {
    const MLimit& R = t.limits[lid];
    rl_limit_desc d;
    d.limit_id = lid;
    d.ns_id = R.ns_id;
    d.varset_id = R.varset_id;
    d.qualified = R.vars.empty() ? 0 : 1;  // counter.rs:108-110
    d.max_value = R.max_value;
    d.window_us = R.seconds * 1000000ull;  // counter.rs:76-78
    return d;
}

}  // namespace

extern "C" {

int rl_matcher_create(rl_matcher** out) {
    if (!out) return RL_FATAL;
    *out = new rl_matcher();
    return RL_OK;
}

void rl_matcher_destroy(rl_matcher* m) { delete m; }

const char* rl_matcher_last_error(rl_matcher* m) { return m ? m->last_error.c_str() : "null matcher"; }

int rl_matcher_last_error_copy(rl_matcher* m, char* out, uint32_t cap) {
    if (!m || !out || !cap) return RL_FATAL;
    std::lock_guard<std::mutex> g(m->err_mu);
    snprintf(out, cap, "%s", m->last_error.c_str());
    return RL_OK;
}

int rl_matcher_add_limit(rl_matcher* m, const char* ns, uint64_t max_value, uint64_t seconds,
                         const char* const* conditions, uint32_t n_cond, const char* const* variables, uint32_t n_var,
                         const char* name, rl_limit_desc* out_desc) {
    return rl_matcher_add_limit_ex(m, ns, max_value, seconds, conditions, n_cond, variables, n_var, name, 0, out_desc, nullptr);
}

int rl_matcher_add_limit_ex(rl_matcher* m, const char* ns, uint64_t max_value, uint64_t seconds,
                            const char* const* conditions, uint32_t n_cond, const char* const* variables, uint32_t n_var,
                            const char* name, int keep_existing, rl_limit_desc* out_desc, int* out_existed) {
    if (!m || !ns || !out_desc || (n_cond && !conditions) || (n_var && !variables)) return RL_FATAL;
    if (out_existed) *out_existed = 0;
    std::unique_lock<std::shared_mutex> lock(m->mu);
    // parse before touching any table: a refused limit leaves the matcher unchanged
    ParsedLimit P;
    std::string err;
    if (!parse_limit(m->dialect, ns, max_value, seconds, conditions, n_cond, variables, n_var, name, nullptr, P, err))
        return mfail(m, "%s", err.c_str());
    const uint32_t lid = place_limit(*m, std::move(P), keep_existing, out_existed);
    m->generation++;
    *out_desc = desc_of(*m, lid);
    return RL_OK;
}

int rl_matcher_set_dialect(rl_matcher* m, uint32_t dialect) {
    if (!m) return RL_FATAL;
    if (dialect != RL_MATCH_DIALECT_TABLE && dialect != RL_MATCH_DIALECT_BOOLEAN) return mfail(m, "unknown dialect %u", dialect);
    std::unique_lock<std::shared_mutex> lock(m->mu);
    m->dialect = dialect;  // the limits already added keep their tests: the image does not change
    return RL_OK;
}

int rl_matcher_set_counter_cap(rl_matcher* m, uint32_t cap) {
    if (!m || cap == 0) return RL_FATAL;
    std::unique_lock<std::shared_mutex> lock(m->mu);
    m->counter_cap = cap;
    m->generation++;
    return RL_OK;
}

// The cap in force (0 for m == NULL).  Library-internal: the RLS service sizes its counter buffers by it.
uint32_t rl_matcher_counter_cap(rl_matcher* m) {
    if (!m) return 0;
    std::shared_lock<std::shared_mutex> lock(m->mu);
    return m->counter_cap;
}

int rl_matcher_delete_limit(rl_matcher* m, uint32_t limit_id) {
    if (!m) return RL_FATAL;
    std::unique_lock<std::shared_mutex> lock(m->mu);
    if (limit_id >= m->limits.size()) return mfail(m, "unknown limit_id %u", limit_id);
    m->limits[limit_id].deleted = true;
    m->generation++;
    return RL_OK;
}

int rl_matcher_namespace_id(rl_matcher* m, const char* ns, uint32_t* out_ns_id) {
    if (!m || !ns || !out_ns_id) return RL_FATAL;
    std::shared_lock<std::shared_mutex> lock(m->mu);
    auto it = m->ns_ids.find(ns);
    if (it == m->ns_ids.end()) return RL_FATAL;
    *out_ns_id = it->second;
    return RL_OK;
}

const char* rl_matcher_limit_name(rl_matcher* m, uint32_t limit_id) {
    if (!m) return nullptr;
    std::shared_lock<std::shared_mutex> lock(m->mu);
    if (limit_id >= m->limits.size() || !m->limits[limit_id].has_name) return nullptr;
    return m->limits[limit_id].name.c_str();
}

int rl_matcher_limit_name_copy(rl_matcher* m, uint32_t limit_id, char* out, uint32_t cap, int* out_has_name) {
    if (!m || !out || !cap) return RL_FATAL;
    std::shared_lock<std::shared_mutex> lock(m->mu);
    out[0] = 0;
    if (out_has_name) *out_has_name = 0;
    if (limit_id >= m->limits.size()) return mfail(m, "unknown limit_id %u", limit_id);
    const MLimit& L = m->limits[limit_id];
    if (!L.has_name) return RL_OK;
    if (L.name.size() + 1 > cap) return mfail(m, "limit name needs %zu bytes", L.name.size() + 1);
    memcpy(out, L.name.c_str(), L.name.size() + 1);
    if (out_has_name) *out_has_name = 1;
    return RL_OK;
}

int rl_matcher_counters(rl_matcher* m, uint32_t ns_id, const rl_binding* binds, uint32_t n_binds, rl_counter* out_ctrs,
                        uint32_t cap, uint32_t* out_n) {
    if (!m || !out_n || (n_binds && !binds) || (cap && !out_ctrs)) return RL_FATAL;
    std::shared_lock<std::shared_mutex> lock(m->mu);
    uint64_t n = 0;
    const int r = match_one(m, ns_id, binds, n_binds, out_ctrs, cap, n, tls_scratch);
    *out_n = (uint32_t)n;
    if (r) return mfail(m, "more than %u counters apply to one request (engine limit %d)", cap, RL_MAX_COUNTERS_PER_REQUEST);
    return RL_OK;
}

int rl_matcher_counters_batch(rl_matcher* m, uint64_t n, const uint32_t* ns_id, const uint32_t* bind_off,
                              const rl_binding* binds, uint32_t* out_ctr_off, rl_counter* out_ctrs, uint64_t cap) {
    if (!m || (n && (!ns_id || !bind_off || !out_ctr_off)) || (cap && !out_ctrs)) return RL_FATAL;
    std::shared_lock<std::shared_mutex> lock(m->mu);
    Scratch& s = tls_scratch;
    uint64_t total = 0;
    if (out_ctr_off) out_ctr_off[0] = 0;
    for (uint64_t i = 0; i < n; i++) {
        uint64_t k = 0;
        const int r = match_one(m, ns_id[i], binds + bind_off[i], bind_off[i + 1] - bind_off[i], out_ctrs + total,
                                cap - total, k, s);
        if (r || total + k > 0xFFFFFFFFull) {
            return mfail(m, "counter capacity %llu exhausted, or more than %d counters apply, at request %llu",
                         (unsigned long long)cap, RL_MAX_COUNTERS_PER_REQUEST, (unsigned long long)i);
        }
        total += k;
        out_ctr_off[i + 1] = (uint32_t)total;
    }
    return RL_OK;
}

// CheckResult::response_header (lib.rs:235-275) of one request into `out`: three NUL-terminated values one after the other
// (X-RateLimit-Limit, -Remaining, -Reset).  Returns the bytes written, 0 when they do not fit in cap, or -1 for an unknown
// limit id.  The caller holds the matcher's lock (shared).  No heap traffic: a batching stage calls it per request.
static int64_t format_headers(const rl_matcher* m, const rl_counter* ctrs, const uint64_t* remaining, const uint64_t* ttl_us, uint32_t n,
                              char* out, uint64_t cap) {
    if (n == 0) {
        if (cap < 3) return 0;
        out[0] = out[1] = out[2] = 0;
        return 3;
    }
    uint32_t small[64];
    std::vector<uint32_t> big;
    uint32_t* order = small;
    if (n > 64) {
        big.resize(n);
        order = big.data();
    }
    for (uint32_t i = 0; i < n; i++) {
        if (ctrs[i].limit_id >= m->limits.size()) return -1;
        // insertion sort by remaining, stable: the most restrictive first (lib.rs:238-242; sort_by is stable)
        uint32_t k = i;
        while (k > 0 && remaining[order[k - 1]] > remaining[i]) {
            order[k] = order[k - 1];
            k--;
        }
        order[k] = i;
    }
    uint64_t w = 0;
    auto put = [&](const char* fmt, unsigned long long a, unsigned long long b) {
        if (w >= cap) return false;
        const int k = snprintf(out + w, cap - w, fmt, a, b);
        if (k < 0 || (uint64_t)k >= cap - w) return false;
        w += (uint64_t)k;
        return true;
    };
    const uint32_t f = order[0];
    if (!put("%llu", m->limits[ctrs[f].limit_id].max_value, 0)) return 0;
    for (uint32_t q = 0; q < n; q++) {  // ", <max>;w=<secs>[;name=\"...\"]" for every counter (lib.rs:244-252)
        const MLimit& L = m->limits[ctrs[order[q]].limit_id];
        if (!put(", %llu;w=%llu", L.max_value, L.seconds)) return 0;
        if (L.has_name) {
            if (w + L.name.size() + 9 >= cap) return 0;
            memcpy(out + w, ";name=\"", 7);
            w += 7;
            for (const char c : L.name) out[w++] = c == '"' ? '\'' : c;
            out[w++] = '"';
        }
    }
    if (w >= cap) return 0;
    out[w++] = 0;
    if (!put("%llu", remaining[f], 0)) return 0;
    if (w >= cap) return 0;
    out[w++] = 0;
    if (!put("%llu", ttl_us[f] / 1000000ull, 0)) return 0;  // Duration::as_secs (lib.rs:268-270)
    if (w >= cap) return 0;
    out[w++] = 0;
    return (int64_t)w;
}

int rl_matcher_counters_batch_ns(rl_matcher* m, uint64_t n, const char* const* ns, const uint32_t* bind_off, const rl_binding* binds,
                                 uint32_t* out_ctr_off, rl_counter* out_ctrs, uint64_t cap, uint8_t* out_status) {
    if (!m || !out_ctr_off || (n && (!ns || !bind_off || !out_status)) || (cap && !out_ctrs)) return RL_FATAL;
    std::shared_lock<std::shared_mutex> lock(m->mu);  // one reader section for the whole range
    Scratch& s = tls_scratch;
    uint64_t total = 0;
    out_ctr_off[0] = 0;
    const char* last_ns = nullptr;  // consecutive requests of one namespace look it up once
    bool last_known = false;
    uint32_t last_id = 0;
    for (uint64_t i = 0; i < n; i++) {
        out_status[i] = 0;
        if (!ns[i]) return mfail(m, "request %llu has no namespace", (unsigned long long)i);
        if (!last_ns || strcmp(ns[i], last_ns) != 0) {
            const auto it = m->ns_ids.find(ns[i]);
            last_ns = ns[i];
            last_known = it != m->ns_ids.end();
            last_id = last_known ? it->second : 0;
        }
        if (!last_known) {
            out_status[i] = 1;  // no limit was ever added for the namespace: nothing applies (lib.rs:434-440)
        } else {
            uint64_t k = 0;
            if (cap - total < m->counter_cap) return mfail(m, "counter capacity %llu exhausted at request %llu", (unsigned long long)cap, (unsigned long long)i);
            if (match_one(m, last_id, binds + bind_off[i], bind_off[i + 1] - bind_off[i], out_ctrs + total, cap - total, k, s) != RL_OK) {
                out_status[i] = 2;  // more counters apply than one request may carry: the request gets none
                k = 0;
            }
            total += k;
        }
        if (total > 0xFFFFFFFFull) return mfail(m, "more than 2^32 counters in one batch");
        out_ctr_off[i + 1] = (uint32_t)total;
    }
    return RL_OK;
}

int rl_matcher_response_headers(rl_matcher* m, const rl_counter* ctrs, const uint64_t* remaining, const uint64_t* ttl_us,
                                uint32_t n, char* out_limit, uint32_t cap_limit, char* out_remaining, uint32_t cap_remaining,
                                char* out_reset, uint32_t cap_reset) {
    if (!m || !out_limit || !out_remaining || !out_reset || !cap_limit || !cap_remaining || !cap_reset ||
        (n && (!ctrs || !remaining || !ttl_us)))
        return RL_FATAL;
    out_limit[0] = out_remaining[0] = out_reset[0] = 0;
    if (n == 0) return RL_OK;
    std::shared_lock<std::shared_mutex> lock(m->mu);
    std::vector<char> text((size_t)cap_limit + 64);
    const int64_t w = format_headers(m, ctrs, remaining, ttl_us, n, text.data(), text.size());
    if (w < 0) return mfail(m, "unknown limit_id in the counters of a response");
    const char* lim = text.data();
    const char* rem = w ? lim + strlen(lim) + 1 : lim;
    const char* rst = w ? rem + strlen(rem) + 1 : lim;
    if (w == 0 || strlen(lim) + 1 > cap_limit || strlen(rem) + 1 > cap_remaining || strlen(rst) + 1 > cap_reset)
        return mfail(m, "header buffer too small for X-RateLimit-Limit (%u bytes given)", cap_limit);
    memcpy(out_limit, lim, strlen(lim) + 1);
    memcpy(out_remaining, rem, strlen(rem) + 1);
    memcpy(out_reset, rst, strlen(rst) + 1);
    return RL_OK;
}

int rl_matcher_response_headers_batch(rl_matcher* m, uint64_t n, const uint32_t* ctr_off, const rl_counter* ctrs, const uint64_t* remaining,
                                      const uint64_t* ttl_us, char* out, uint64_t cap, uint64_t* out_off, uint64_t* out_len) {
    if (!m || !out_off || !out_len || (n && (!ctr_off || !ctrs || !remaining || !ttl_us)) || (cap && !out)) return RL_FATAL;
    std::shared_lock<std::shared_mutex> lock(m->mu);  // one reader section for the whole range
    uint64_t w = 0;
    bool fits = true;
    out_off[0] = 0;
    char scratch[4096];
    for (uint64_t i = 0; i < n; i++) {
        const uint32_t o = ctr_off[i], k = ctr_off[i + 1] - o;
        int64_t got = fits ? format_headers(m, ctrs + o, remaining + o, ttl_us + o, k, out + w, cap - w) : 0;
        if (got < 0) return mfail(m, "unknown limit_id in the counters of request %llu", (unsigned long long)i);
        if (got == 0) {  // does not fit (any more): keep measuring so that *out_len tells the caller what to bring
            fits = false;
            std::vector<char> big;
            char* tmp = scratch;
            uint64_t tcap = sizeof scratch;
            while ((got = format_headers(m, ctrs + o, remaining + o, ttl_us + o, k, tmp, tcap)) == 0) {
                big.resize(tcap * 4);
                tmp = big.data();
                tcap = big.size();
            }
            if (got < 0) return mfail(m, "unknown limit_id in the counters of request %llu", (unsigned long long)i);
        }
        w += (uint64_t)got;
        out_off[i + 1] = w;
    }
    *out_len = w;
    return fits ? RL_OK : mfail(m, "header text needs %llu bytes", (unsigned long long)w);
}

uint64_t rl_matcher_generation(rl_matcher* m) {
    if (!m) return 0;
    std::shared_lock<std::shared_mutex> lock(m->mu);
    return m->generation;
}

int rl_matcher_image(rl_matcher* m, uint32_t* out, uint64_t cap_words, uint64_t* out_words, uint64_t* out_generation) {
    if (!m || !out_words || (cap_words && !out)) return RL_FATAL;
    std::shared_lock<std::shared_mutex> lock(m->mu);
    std::vector<uint32_t> w(RL_IMG_HDR_WORDS, 0);
    std::string arena;
    auto put_str = [&](const std::string& x) {
        const uint32_t o = (uint32_t)arena.size();
        arena += x;
        return o;
    };
    auto table_mask = [](size_t n) {
        size_t cap = 16;
        while (cap < 2 * n) cap *= 2;
        return (uint32_t)(cap - 1);
    };
    // namespaces: id -> string, then the open-addressed table
    const uint32_t n_ns = (uint32_t)m->ns_limits.size();
    std::vector<const std::string*> ns_of(n_ns, nullptr);
    for (const auto& kv : m->ns_ids) ns_of[kv.second] = &kv.first;
    const uint32_t ns_mask = table_mask(n_ns);
    w[RL_IMG_H_NS_TAB] = (uint32_t)w.size();
    w.resize(w.size() + ns_mask + 1, RL_IMG_EMPTY);
    w[RL_IMG_H_NS_STR] = (uint32_t)w.size();
    for (uint32_t id = 0; id < n_ns; id++) {
        const std::string& x = *ns_of[id];
        w.push_back(put_str(x));
        w.push_back((uint32_t)x.size());
        uint32_t* tab = w.data() + w[RL_IMG_H_NS_TAB];
        uint64_t p = rl_img_hash(RL_IMG_NS_SEED, (const uint8_t*)x.data(), (uint32_t)x.size()) & ns_mask;
        while (tab[p] != RL_IMG_EMPTY) p = (p + 1) & ns_mask;
        tab[p] = id;
    }
    // per namespace, its live limits in counter output order
    w[RL_IMG_H_NS_LIM_OFF] = (uint32_t)w.size();
    w.resize(w.size() + n_ns + 1, 0);
    w[RL_IMG_H_NS_LIMS] = (uint32_t)w.size();
    for (uint32_t id = 0; id < n_ns; id++) {
        w[w[RL_IMG_H_NS_LIM_OFF] + id] = (uint32_t)(w.size() - w[RL_IMG_H_NS_LIMS]);
        for (const uint32_t lid : m->ns_limits[id])
            if (!m->limits[lid].deleted) w.push_back(lid);
    }
    w[w[RL_IMG_H_NS_LIM_OFF] + n_ns] = (uint32_t)(w.size() - w[RL_IMG_H_NS_LIMS]);
    // slots
    const uint32_t n_slots = (uint32_t)m->slots.keys.size();
    const uint32_t slot_mask = table_mask(n_slots);
    w[RL_IMG_H_SLOT_TAB] = (uint32_t)w.size();
    w.resize(w.size() + slot_mask + 1, RL_IMG_EMPTY);
    w[RL_IMG_H_SLOT_KEY] = (uint32_t)w.size();
    for (uint32_t s = 0; s < n_slots; s++) {
        const SlotKey& k = m->slots.keys[s];
        w.push_back(k.desc);
        w.push_back(put_str(k.key));
        w.push_back((uint32_t)k.key.size());
        uint32_t* tab = w.data() + w[RL_IMG_H_SLOT_TAB];
        uint64_t p = rl_img_hash(k.desc, (const uint8_t*)k.key.data(), (uint32_t)k.key.size()) & slot_mask;
        while (tab[p] != RL_IMG_EMPTY) p = (p + 1) & slot_mask;
        tab[p] = s;
    }
    // limits, their tests, the tests' atoms and the limits' variables
    const uint32_t n_limits = (uint32_t)m->limits.size();
    std::vector<uint32_t> tests, atoms, vars;
    w[RL_IMG_H_LIMS] = (uint32_t)w.size();
    for (uint32_t lid = 0; lid < n_limits; lid++) {
        const MLimit& L = m->limits[lid];
        w.push_back((uint32_t)(tests.size() / 4));
        w.push_back((uint32_t)L.tests.size());
        w.push_back((uint32_t)(vars.size() / 3));
        w.push_back((uint32_t)L.var_slots.size());
        w.push_back(L.varset_id);
        for (const Test& t : L.tests) {
            tests.push_back(t.slot);
            tests.push_back((uint32_t)(atoms.size() / 3) << 3 | (uint32_t)t.atoms.size());
            tests.push_back((uint32_t)t.table);
            tests.push_back((uint32_t)(t.table >> 32));
            for (const Atom& a : t.atoms) {
                atoms.push_back(a.op);
                if (a.op != RL_ATOM_IN) {
                    atoms.push_back(put_str(a.lits[0]));
                    atoms.push_back((uint32_t)a.lits[0].size());
                    continue;
                }
                atoms.push_back((uint32_t)arena.size());
                atoms.push_back((uint32_t)a.lits.size());
                for (const std::string& l : a.lits) {
                    const uint32_t n = (uint32_t)l.size();
                    const char le[4] = {(char)n, (char)(n >> 8), (char)(n >> 16), (char)(n >> 24)};
                    arena.append(le, 4);
                    arena += l;
                }
            }
        }
        for (size_t j = 0; j < L.var_slots.size(); j++) {
            vars.push_back(L.var_slots[j]);
            vars.push_back(put_str(L.vars[j]));
            vars.push_back((uint32_t)L.vars[j].size());
        }
    }
    if (atoms.size() / 3 >= (1u << 29)) return mfail(m, "more than 2^29 value atoms in one matcher image");
    w[RL_IMG_H_TESTS] = (uint32_t)w.size();
    w.insert(w.end(), tests.begin(), tests.end());
    w[RL_IMG_H_ATOMS] = (uint32_t)w.size();
    w.insert(w.end(), atoms.begin(), atoms.end());
    w[RL_IMG_H_VARS] = (uint32_t)w.size();
    w.insert(w.end(), vars.begin(), vars.end());
    w[RL_IMG_H_ARENA] = (uint32_t)w.size();
    w[RL_IMG_H_ARENA_BYTES] = (uint32_t)arena.size();
    const size_t arena_words = (arena.size() + 3) / 4;
    w.resize(w.size() + arena_words, 0);
    if (!arena.empty()) memcpy(w.data() + w[RL_IMG_H_ARENA], arena.data(), arena.size());
    w[RL_IMG_H_MAGIC] = RL_IMG_MAGIC;
    w[RL_IMG_H_N_NS] = n_ns;
    w[RL_IMG_H_NS_MASK] = ns_mask;
    w[RL_IMG_H_N_SLOTS] = n_slots;
    w[RL_IMG_H_SLOT_MASK] = slot_mask;
    w[RL_IMG_H_N_LIMITS] = n_limits;
    w[RL_IMG_H_COUNTER_CAP] = m->counter_cap;
    *out_words = w.size();
    if (out_generation) *out_generation = m->generation;
    if (w.size() > cap_words) return RL_FATAL;
    memcpy(out, w.data(), w.size() * sizeof(uint32_t));
    return RL_OK;
}

}  // extern "C"

bool rl_matcher_ns_limit_records(rl_matcher* m, const std::string& ns, std::vector<RlLimitRecord>& out) {
    out.clear();
    if (!m) return false;
    std::shared_lock<std::shared_mutex> lock(m->mu);
    const auto it = m->ns_ids.find(ns);
    if (it == m->ns_ids.end()) return false;
    for (const uint32_t lid : m->ns_limits[it->second]) {
        const MLimit& L = m->limits[lid];
        if (L.deleted) continue;
        RlLimitRecord r;
        r.limit_id = lid;
        r.varset_id = L.varset_id;
        r.max_value = L.max_value;
        r.seconds = L.seconds;
        r.has_name = L.has_name;
        r.name = L.name;
        r.has_id = L.has_id;
        r.id = L.id;
        r.conditions = L.conds;
        r.variables = L.vars;
        out.push_back(std::move(r));
    }
    return true;
}

int rl_matcher_configure(rl_matcher* m, const rl_limit_spec* specs, uint32_t n, uint32_t max_limits_per_ns, bool dry_run,
                         RlConfigurePlan& plan, const std::function<int(RlConfigurePlan&)>& apply) {
    plan = RlConfigurePlan();
    if (!m || (n && !specs)) return RL_FATAL;
    std::unique_lock<std::shared_mutex> lock(m->mu);
    const auto refuse = [&](uint32_t i, std::string why) {
        plan.refused = i;
        plan.error = rl_format("entry %u: %s", i, why.c_str());
        return RL_FATAL;
    };
    // 1. every entry parsed in the dialect in force; the first of two entries with one identity wins (HashSet::insert)
    std::vector<ParsedLimit> parsed(n);
    std::vector<uint8_t> first(n, 0);
    std::map<std::string, uint32_t> wanted;  // identity -> entry
    std::unordered_map<std::string, uint32_t> per_ns;
    const uint32_t cap = std::min(max_limits_per_ns, m->counter_cap);
    for (uint32_t i = 0; i < n; i++) {
        const rl_limit_spec& x = specs[i];
        if (!x.ns || (x.n_cond && !x.conditions) || (x.n_var && !x.variables)) return refuse(i, "null namespace or expression list");
        std::string err;
        if (!parse_limit(m->dialect, x.ns, x.max_value, x.seconds, x.conditions, x.n_cond, x.variables, x.n_var, x.name, x.id, parsed[i], err))
            return refuse(i, err);
        if (!wanted.emplace(parsed[i].ident, i).second) continue;
        first[i] = 1;
        if (++per_ns[parsed[i].L.ns] > cap)
            return refuse(i, rl_format("namespace %s would hold more than %u limits, the counters one request may carry", x.ns, cap));
    }
    // 2. staged on a copy of the tables: live limits absent from the new set are deleted, kept ones stay where they are,
    // added ones follow in the given order
    MTables t = *m;
    for (uint32_t lid = 0; lid < t.limits.size(); lid++) {
        MLimit& L = t.limits[lid];
        if (L.deleted) continue;
        if (wanted.count(identity_of(L))) continue;
        L.deleted = true;
        plan.deleted.push_back(lid);
    }
    for (uint32_t i = 0; i < n; i++) {
        if (!first[i]) continue;
        ParsedLimit& P = parsed[i];
        const auto it = t.by_identity.find(P.ident);
        const MLimit* E = it == t.by_identity.end() ? nullptr : &t.limits[it->second];
        if (E && !E->deleted && E->max_value == P.L.max_value && E->has_name == P.L.has_name && E->name == P.L.name) {
            plan.kept++;  // update_limit compares max_value and name only: the old id stays too
            continue;
        }
        const bool update = E && !E->deleted;
        const uint64_t old_max = update ? E->max_value : 0;
        const uint32_t lid = place_limit(t, std::move(P), 0, nullptr);
        plan.set.push_back(desc_of(t, lid));
        plan.set_entry.push_back(i);
        plan.set_added.push_back(update ? 0 : 1);
        plan.old_max.push_back(old_max);
        (update ? plan.updated : plan.added)++;
    }
    if (dry_run) return RL_OK;
    // 3. the engine (the caller's apply), then the matcher in one step
    const int r = apply ? apply(plan) : RL_OK;
    if (r != RL_OK) return r;
    static_cast<MTables&>(*m) = std::move(t);
    m->generation++;
    return RL_OK;
}

extern "C" {

void rl_counter_key(const char* const* sources, const char* const* values, uint32_t n, uint64_t* key_lo, uint64_t* key_hi) {
    *key_lo = *key_hi = 0;
    if (n == 0) return;
    std::vector<uint32_t> order(n);
    for (uint32_t i = 0; i < n; i++) order[i] = i;
    std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return strcmp(sources[a], sources[b]) < 0; });
    KeyDigest d;
    for (const uint32_t i : order) {
        d.str(sources[i], strlen(sources[i]));
        d.str(values[i], strlen(values[i]));
    }
    d.finish(*key_lo, *key_hi);
}

}  // extern "C"
