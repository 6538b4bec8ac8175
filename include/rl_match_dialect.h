/* rl_match_dialect.h — the condition grammar of a matcher (include/rl_match.h, which includes this header).
 *
 * RL_MATCH_DIALECT_TABLE (every matcher's default) accepts `operand ==|!= 'literal'` conditions only;
 * RL_MATCH_DIALECT_BOOLEAN also accepts boolean formulas over one operand (&&, ||, !, in, startsWith, endsWith, contains)
 * and positive presence tests as top-level conjuncts.  rl_match.h states both grammars.
 */
#ifndef RL_MATCH_DIALECT_H
#define RL_MATCH_DIALECT_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RL_MATCH_DIALECT_TABLE 0u
#define RL_MATCH_DIALECT_BOOLEAN 1u

struct rl_matcher;
/* The dialect in which the matcher's LATER rl_matcher_add_limit / _ex calls parse their conditions.  Limits already
 * added keep their meaning (the device image does not change); variables parse the same in both.  RL_FATAL for an
 * unknown dialect. */
int rl_matcher_set_dialect(struct rl_matcher *m, uint32_t dialect);

#ifdef __cplusplus
}
#endif
#endif /* RL_MATCH_DIALECT_H */
