// Host side of the rollout kernels' dispatch, shared by K1 (rollout.cu) and K1-TC (rollout_tc.cu): the task a launch flies,
// the kernel variant a checked launch description selects, and the list of the variants the kernels are instantiated for.
#pragma once
#include <type_traits>

#include "../../include/serl_b200.h"

// The PH-LAB task of a rollout and its actor's observation and action widths
struct RolloutTask {
    bool inc;                  // incremental control (SERL_ROLLOUT_INCREMENTAL)
    bool sym;                  // symmetric control (SERL_ROLLOUT_SYMMETRIC); neither: attitude control
    int obs, act;
};
constexpr RolloutTask TASK_ATTITUDE = {false, false, 7, 3};
constexpr RolloutTask TASK_INCREMENTAL = {true, false, 10, 3};
constexpr RolloutTask TASK_SYMMETRIC = {false, true, 2, 1};

static inline RolloutTask task_of_flags(int32_t flags)
{
    return (flags & SERL_ROLLOUT_INCREMENTAL) ? TASK_INCREMENTAL : (flags & SERL_ROLLOUT_SYMMETRIC) ? TASK_SYMMETRIC : TASK_ATTITUDE;
}

// the task whose widths the shape has (for callers without flags), or nullptr
static inline const RolloutTask* task_of_shape(const serl_actor_shape& sh)
{
    for (const RolloutTask* t : {&TASK_ATTITUDE, &TASK_INCREMENTAL, &TASK_SYMMETRIC})
        if (sh.state_dim == t->obs && sh.action_dim == t->act) return t;
    return nullptr;
}

// calls f(S, A) with the task's observation and action widths as std::integral_constant
template <typename F>
void visit_task(const RolloutTask& t, F&& f)
{
    using std::integral_constant;
    if (t.inc) f(integral_constant<int, TASK_INCREMENTAL.obs>(), integral_constant<int, TASK_INCREMENTAL.act>());
    else if (t.sym) f(integral_constant<int, TASK_SYMMETRIC.obs>(), integral_constant<int, TASK_SYMMETRIC.act>());
    else f(integral_constant<int, TASK_ATTITUDE.obs>(), integral_constant<int, TASK_ATTITUDE.act>());
}

// The kernel variant of a launch: the rollout kernels' template flags GUST, TRACK, PER_ACTOR and the task (INC, SYM)
struct RolloutVariant {
    bool gust, track, per_actor;
    RolloutTask task;
};

// The variant a checked launch description flies:
//   - a launch with d_track flies its task's tracking variant, which carries the gust schedule and reads no per-actor rows;
//   - any other launch flies (task, SERL_ROLLOUT_GUST, SERL_ROLLOUT_PER_ACTOR_REFS).
static inline RolloutVariant rollout_variant(const serl_rollout_desc& d, const RolloutTask& task)
{
    if (d.d_track) return {true, true, false, task};
    return {(d.flags & SERL_ROLLOUT_GUST) != 0, false, (d.flags & SERL_ROLLOUT_PER_ACTOR_REFS) != 0, task};
}

// one instantiated variant as compile-time values
template <bool G, bool T, bool P, bool I, bool S>
struct RolloutFlags {
    static constexpr bool GUST = G, TRACK = T, PER_ACTOR = P, INC = I, SYM = S;
};

template <bool G, bool T, bool P, bool I, bool S, typename F>
bool visit_if(const RolloutVariant& v, F& f)
{
    if (v.gust != G || v.track != T || v.per_actor != P || v.task.inc != I || v.task.sym != S) return false;
    f(RolloutFlags<G, T, P, I, S>());
    return true;
}

// The 11 variants every rollout kernel is instantiated for: when v is one of them, calls f(RolloutFlags<...>()) and returns
// true.  The evaluation suite's tracking launches fly gust envs, so tracking carries the gust schedule; no tracking launch
// takes per-actor refs; incremental control flies the nominal build only and symmetric control takes gust envs in the suite
// only, so neither has a gust training instantiation.  check_desc refuses every launch outside the list, which makes the
// visit total on the descriptors that reach a kernel.
template <typename F>
bool visit_rollout_variant(const RolloutVariant& v, F&& f)
{
    //              GUST   TRACK  PER_ACTOR INC  SYM
    return visit_if<false, false, false, false, false>(v, f) ||      // attitude control
           visit_if<true,  false, false, false, false>(v, f) ||
           visit_if<false, false, true,  false, false>(v, f) ||
           visit_if<true,  false, true,  false, false>(v, f) ||
           visit_if<true,  true,  false, false, false>(v, f) ||
           visit_if<false, false, false, true,  false>(v, f) ||      // incremental control
           visit_if<false, false, true,  true,  false>(v, f) ||
           visit_if<true,  true,  false, true,  false>(v, f) ||
           visit_if<false, false, false, false, true >(v, f) ||      // symmetric control
           visit_if<false, false, true,  false, true >(v, f) ||
           visit_if<true,  true,  false, false, true >(v, f);
}
