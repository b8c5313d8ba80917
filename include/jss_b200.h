/*
 * jss_b200.h -- C-ABI of the H100-native batched job-shop environment.
 *
 * The reference (prosysscience/JSSEnv) has NO FFI layer: its boundary is the
 * Python object protocol of `JssEnv` (JSSEnv/envs/jss_env.py:14).  Each entry
 * point below names the reference interface it replaces (file:line relative to
 * the reference tree).  The Python mirror of that interface lives in
 * jssenv_b200/ (JssEnv / JssVecEnv / dispatching) and binds these symbols with
 * ctypes; INTEGRATION.md shows the stub a reference maintainer would add.
 *
 * Conventions
 *   - plain pointers and sizes only; no C++/torch types cross this boundary;
 *   - every call returns JSS_OK (0) or a negative JSS_ERR_* code and never throws;
 *     jss_last_error() gives the message for the handle (or for creation if NULL);
 *   - the library owns all device memory; jss_get_buffers() exposes device
 *     pointers that stay valid until jss_destroy(); callers wrap them zero-copy;
 *   - all work is enqueued on the `stream` argument (a cudaStream_t passed as
 *     void*; NULL = the legacy default stream) and is asynchronous unless the
 *     call says otherwise; a handle is bound to ONE device and is not thread-safe
 *     (multi-GPU = one process/handle per GPU);
 *   - there is NO CPU fallback: without a CUDA device jss_create() fails with
 *     JSS_ERR_NO_DEVICE.
 *
 * Batched semantics (N independent envs; env i runs instance env_to_inst[i]):
 *   action a in [0, J_i)  allocate job a            (jss_env.py:441-481)
 *   action a == J_i       no-op / wait              (jss_env.py:419-440)
 *   action JSS_ACTION_SKIP     leave env i untouched this call
 *   action JSS_ACTION_ADVANCE  raw increase_time_step() (jss_env.py:495-637),
 *                              the hook tests/test_solutions.py:66 calls directly
 *   Reference exceptions become a per-env sticky error bit (JSS_FLAG_ERROR) and
 *   the env is left unchanged for that call: job action that is not legal,
 *   finished job (IndexError jss_env.py:444), no-op with no pending event
 *   (IndexError jss_env.py:517), out-of-range action.
 *   A done env is frozen (its terminal observation stays readable) until it is
 *   reset; with JSS_CREATE_AUTO_RESET the next jss_step() on it performs the
 *   reset instead (reward 0, done 0).
 */
#ifndef JSS_B200_H
#define JSS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define JSS_ABI_VERSION 3

/* limits of the one-warp-per-env kernels */
#define JSS_MAX_JOBS 256
#define JSS_MAX_MACHINES 32
#define JSS_MAX_DURATION 2047
#define JSS_MAX_BEAM_WIDTH 32   /* beams per env of jss_beam_search() */

/* return codes */
#define JSS_OK 0
#define JSS_ERR_INVALID (-1)     /* bad argument */
#define JSS_ERR_NO_DEVICE (-2)   /* no CUDA device / wrong architecture */
#define JSS_ERR_CUDA (-3)        /* a CUDA runtime call failed (see jss_last_error) */
#define JSS_ERR_UNSUPPORTED (-4) /* instance exceeds JSS_MAX_*, or has a zero-length op (the reference cannot finish such an
                                    episode either: jss_env.py:529 never sees the op as completed) */
#define JSS_ERR_STATE (-5)       /* call order violated (e.g. step before load/assign) */

/* special actions */
#define JSS_ACTION_SKIP (-1)
#define JSS_ACTION_ADVANCE (-2)

/* jss_create flags */
#define JSS_CREATE_AUTO_RESET 1u      /* step() on a done env resets it */
#define JSS_CREATE_RECORD_SOLUTION 2u /* keep solution[N][Jmax][Mmax] start times (jss_env.py:163,454) */
#define JSS_CREATE_HOST_MIRROR 4u     /* small batches (the single-env facade): action_mask, real_obs, the scalar records,
                                         the x_* arrays and an action slot live in ONE pinned, device-mapped host block --
                                         the kernels write results straight into host memory, no copies per transition */

/* per-env flag bits (jss_buffers.flags_done >> 8) */
#define JSS_FLAG_DONE 1u        /* _is_done() (jss_env.py:639-653) */
#define JSS_FLAG_ERROR 2u       /* sticky until reset */
#define JSS_FLAG_NOOP_LEGAL 4u  /* legal_actions[J] */

/* dispatching rules (JSSEnv/dispatching.py); RANDOM = masked-uniform policy
 * (README.md:58-60) */
#define JSS_RULE_RANDOM 0
#define JSS_RULE_SPT 1   /* dispatching.py:92-116  */
#define JSS_RULE_FIFO 2  /* dispatching.py:133-156 */
#define JSS_RULE_MWR 3   /* dispatching.py:173-199 */
#define JSS_RULE_LWR 4   /* dispatching.py:216-242 */
#define JSS_RULE_MOR 5   /* dispatching.py:259-283 */
#define JSS_RULE_LOR 6   /* dispatching.py:300-324 */
#define JSS_RULE_CR 7    /* dispatching.py:365-408 */
#define JSS_NUM_RULES 8

/* jss_policy coin modes for the rules' "10 % wait" draw (dispatching.py:113) */
#define JSS_COIN_DEVICE 0 /* counter RNG: wait iff hash(seed, env, step) < 0.1 * 2^32 */
#define JSS_COIN_NEVER 1  /* never wait; caller reads JSS_FLAG_NOOP_LEGAL and decides (host np.random) */

typedef struct jss_handle jss_t;

/* Device pointers owned by the library (jss_get_buffers).
 * Layout: row-major, env-major.  J = jobs_max, M = machines_max of the batch. */
typedef struct jss_buffers {
    int32_t n_envs;
    int32_t jobs_max;       /* J */
    int32_t machines_max;   /* M */
    int32_t mask_stride;    /* bytes per action_mask row (>= J+1, multiple of 4) */
    uint8_t *action_mask;   /* [N][mask_stride]; bytes 0..J_i = legal_actions of env i (jss_env.py:133) */
    float *real_obs;        /* [N][J][7] fp32 (jss_env.py:102-111, 132).  Invariant: at the entry of every
                               step, real_obs[i] equals the observation of env i's state block, unless the handle
                               has it marked stale (then the step re-emits it first).  The uniform-batch step
                               kernels rely on it: they rewrite only the 32-byte sectors of a row the step changed.
                               Every path that writes a state block emits the row or marks it stale; a caller must
                               treat real_obs as read-only. */
    int32_t scalar_stride;  /* bytes between consecutive envs in the five per-env scalar arrays below
                               (they are fields of one 16-byte record per env, written with one store) */
    int32_t host_mirror;    /* 1: the output pointers below are host-readable (JSS_CREATE_HOST_MIRROR) */
    float *reward;          /* [N] scaled reward (jss_env.py:483-493)              */
    int32_t *reward_raw;    /* [N] reward before scaling; -hole for ACTION_ADVANCE */
    uint8_t *done;          /* [N] 0/1 (low byte of flags_done)                    */
    int32_t *time;          /* [N] current_time_step (makespan once done)          */
    uint32_t *flags_done;   /* [N] (JSS_FLAG_* << 8) | done                        */
    int32_t *solution;      /* [N][J][M] or NULL (JSS_CREATE_RECORD_SOLUTION)      */
    /* per-env episode statistics, updated when an episode ends */
    int32_t *episode_count;     /* [N] finished episodes               */
    int32_t *last_makespan;     /* [N] makespan of the last finished episode (jss_env.py:650) */
    int32_t *last_return;       /* [N] raw return of the last finished episode */
    /* canonical (decoded) state, filled by jss_export_state only */
    int32_t *x_todo;        /* [N][J] todo_time_step_job                  */
    int32_t *x_tufco;       /* [N][J] time_until_finish_current_op_jobs   */
    int32_t *x_idle_last;   /* [N][J] idle_time_jobs_last_op              */
    int32_t *x_total_idle;  /* [N][J] total_idle_time_jobs                */
    int32_t *x_col4;        /* [N][J] numerator of real_obs[:,4]; max_time_op encodes 1.0 */
    int32_t *x_tuam;        /* [N][M] time_until_available_machine        */
    uint8_t *x_legal;       /* [N][J] legal_actions[:-1]                  */
    uint8_t *x_blocked;     /* [N][J] action_illegal_no_op                */
    int32_t *mirror_actions; /* [N] action slot inside the host block (JSS_CREATE_HOST_MIRROR), else NULL */
} jss_buffers;

/* number of int64 slots jss_stats() writes */
#define JSS_STATS_LEN 8
/* [0] finished episodes  [1] env steps executed  [2] sum of makespans
 * [3] min makespan (INT64_MAX if none)  [4] max makespan  [5] sum of raw returns
 * [6] envs currently done  [7] envs with the error bit set */

/* --- lifetime ---------------------------------------------------------- */

/* Replaces JssEnv.__init__ (jss_env.py:27-119) for a batch of n_envs envs on CUDA
 * device `device`.  `env_id_base` is the global index of env 0 (multi-GPU
 * shards: rank r passes r * n_envs so RNG streams do not depend on the world
 * size). */
int jss_create(jss_t **out, int device, int n_envs, uint32_t flags, uint64_t env_id_base);
void jss_destroy(jss_t *h);
const char *jss_last_error(const jss_t *h);
int jss_abi_version(void);

/* Replaces the instance parse (jss_env.py:72-95): n_inst instances, instance k
 * has jobs[k] x machines[k] operations stored row-major at
 * machine[offsets[k] ...] / duration[offsets[k] ...] (host pointers). */
int jss_load_instances(jss_t *h, int n_inst, const int32_t *jobs, const int32_t *machines,
                       const int64_t *offsets, const int32_t *machine, const int32_t *duration);

/* env i runs instance env_to_inst[i] (host pointer, n_envs entries); allocates
 * all device buffers and resets every env.  Must follow jss_load_instances.
 * Synchronous: returns once its device work has completed, so the batch may be
 * stepped at once on any stream. */
int jss_assign(jss_t *h, const int32_t *env_to_inst);

int jss_get_buffers(jss_t *h, jss_buffers *out);

/* derived per-instance scalars (jss_env.py:86-89): out[0]=max_time_op,
 * out[1]=max_time_jobs, out[2]=sum_op */
int jss_instance_scalars(jss_t *h, int inst, int64_t out[3]);

/* --- hot path ------------------------------------------------------------ */

/* Replaces reset() (jss_env.py:145-181).  env_mask_dev: device u8[N], nonzero =
 * reset that env; NULL = reset all. */
int jss_reset(jss_t *h, const uint8_t *env_mask_dev, void *stream);

/* Replaces step() (jss_env.py:403-481) incl. increase_time_step (495-637),
 * _prioritization_non_final (183-254), _check_no_op (256-401), _reward_scaler
 * (483-493), _is_done (639-653), _get_current_state_representation (121-134).
 * actions_dev: device int32[N]. */
int jss_step(jss_t *h, const int32_t *actions_dev, void *stream);

/* jss_step() + jss_export_state() in ONE launch (generic kernel): the latency path of the single-env facade, which
 * needs the decoded state after every transition to serve the reference's attribute surface. */
int jss_step_export(jss_t *h, const int32_t *actions_dev, void *stream);

/* Replaces DispatchingRule.__call__ (dispatching.py:92-408) / the masked-random
 * sampler (README.md:58-60).  Writes device int32[N] actions.  `step_index` is
 * the RNG counter (callers increment it per decision). */
int jss_policy(jss_t *h, int rule, int coin_mode, uint64_t seed, uint64_t step_index,
               int32_t *actions_dev, void *stream);

/* Replaces CriticalRatio.__init__(due_date_factor) (dispatching.py:337-349): the factor JSS_RULE_CR multiplies a
 * job's total processing time with to get its due date (dispatching.py:357-360).  Default 1.5 like the reference;
 * applies to every later jss_policy / jss_step_sample / jss_rollout with JSS_RULE_CR on this handle. */
int jss_set_cr_due_date_factor(jss_t *h, double factor);

/* jss_step() fused with jss_policy() for the NEXT decision: applies actions_dev, then
 * writes every env's next action (chosen by `rule` on the new state, RNG counter
 * `step_index`) to next_actions_dev, in one launch.  The two buffers may alias. */
int jss_step_sample(jss_t *h, const int32_t *actions_dev, int rule, int coin_mode, uint64_t seed,
                    uint64_t step_index, int32_t *next_actions_dev, void *stream);

/* Step a batch from policy logits (the action_mask-restricted categorical draw of README.md:84-97, driven by a
 * network instead of np.random.choice): chooses every env's action from its logits row, then applies it exactly as
 * jss_step() would, in one launch, and writes the chosen actions and their log-probabilities.
 *   logits_dev: device fp32 [N][ld], ld >= jobs_max + 1, unit column stride.  Columns 0..J_i-1 of env i's row are
 *     its jobs, column J_i its no-op (the columns of its action_mask row); columns past J_i are never read.
 *   Candidates: the actions legal in the env's current state (the action_mask the caller's network saw).  Logits of
 *     illegal actions are ignored whatever their value, NaN and +-inf included.
 *   Draw: Gumbel-max, a = argmax over legal a of (logit[a] - mx) + g[a], mx the largest legal logit,
 *     g = -log(-log u[a]), ties to the lowest index, with u[a] = ((H(h_env, a) >> 8) + 0.5) * 2^-24, H = jss_hash_env
 *     and h_env = jss_hash3 of (seed, env_id_base + i, step_index) (jss_rng.h): replayable on the host and independent
 *     of sharding.  Computed in fp32.  The key is max-subtracted so that the draw follows log_prob at any magnitude:
 *     adding one constant to every legal logit changes neither the draw nor log_prob wherever it leaves their
 *     differences exact, and tied logits at 1e30 are drawn uniformly.  Earlier builds keyed on logit[a] + g[a]: for
 *     a given seed, the draw now differs from theirs only where the fp32 rounding of that sum decided it (large
 *     logits, near ties).  The ABI is unchanged.
 *   log_prob_out_dev[i] = (logit[a] - mx) - log sum exp(legal logits - mx), fp32.
 *   Special cases (as env_select_action / jss_step):
 *     done env: frozen, or reset under JSS_CREATE_AUTO_RESET, as by jss_step(); writes action 0, log_prob 0;
 *     only the no-op legal: action J_i, log_prob 0 (its logit is not read);
 *     bad logits (a legal logit NaN or +inf, or every legal logit -inf): the env gets the sticky JSS_FLAG_ERROR bit
 *       and is left unchanged, like an illegal action; writes action JSS_ACTION_SKIP, log_prob NaN;
 *     no legal action at all (not reachable from reset; an imported state): env untouched, JSS_ACTION_SKIP, NaN.
 *   actions_out_dev: device int32[N] (required); log_prob_out_dev: device fp32[N], NULL skips that store.
 *   Returns JSS_ERR_INVALID for a NULL logits_dev / actions_out_dev or ld < jobs_max + 1. */
int jss_step_logits(jss_t *h, const float *logits_dev, int64_t ld, uint64_t seed, uint64_t step_index,
                    int32_t *actions_out_dev, float *log_prob_out_dev, void *stream);

/* jss_step_logits() that records the transition straight into the caller's rollout slot (what an on-policy collector
 * keeps per step), in the same one launch: the draw, the RNG, the special cases, the JSS_ERR_INVALID rules and
 * everything the env keeps (state, action_mask, scalar records, statistics, solution) are exactly those of
 * jss_step_logits(), but the observation goes to obs_out_dev instead of real_obs.
 *   obs_out_dev [N][jobs_max][7] fp32, mask_out_dev [N][mask_stride] u8, scalars_out_dev [N][4] int32 (the 16-byte
 *     records): the layouts of real_obs, action_mask and the scalar records.  Every env's row is written, also for an
 *     env the call left unchanged (a frozen done env, an env that got the error bit): the observation and mask rows
 *     are what real_obs / action_mask would hold after jss_step_logits(), and the record is too, except that an
 *     unchanged env gets reward 0 and raw reward 0 (as in jss_rollout_traj).  Row bytes past J_i are not written.
 *   The three pointers are required and 16-byte aligned (JSS_ERR_INVALID otherwise); log_prob_out_dev may be NULL.
 *   real_obs is not written and becomes stale: jss_refresh_obs() rewrites it.  Every entry point other than this one,
 *   jss_export_state, jss_policy and jss_stats does that by itself before its first launch, so each keeps its
 *   meaning; only a caller reading real_obs directly after a recording step needs the explicit call.
 * Bytes per ta80 env-step: 5 724 against 5 604 for jss_step_logits() (the mask row and the record are written twice),
 * where jss_step_logits() followed by copies of the observation, mask and record moves about 11 400.  Measured on an
 * H100 SXM 80 GB HBM3 at a 700 W power limit (ta80, N = 65 536, median of three runs): 164.4 us per step, against
 * 316.4 us for jss_step_logits() plus torch copies into the same buffers and 160.1 us for jss_step_logits() alone
 * (DESIGN.md section 4). */
int jss_step_logits_record(jss_t *h, const float *logits_dev, int64_t ld, uint64_t seed, uint64_t step_index,
                           int32_t *actions_out_dev, float *log_prob_out_dev, float *obs_out_dev, uint8_t *mask_out_dev,
                           int32_t *scalars_out_dev, void *stream);

/* Step a batch greedily or epsilon-greedily from action scores (greedy evaluation of a trained policy, epsilon-greedy collection
 * for a value-based agent): chooses every env's action from its row of scores, then applies it exactly as jss_step()
 * would, in one launch, and writes the chosen actions and their log-probabilities under the epsilon-greedy policy.
 *   scores_dev: logits or Q-values, with the layout, ld rule and columns of jss_step_logits(); only legal columns are
 *     read, and scores of illegal actions are ignored whatever their value, NaN and +-inf included.
 *   Bad scores: the rule of jss_step_logits() (a legal score NaN or +inf, or every legal score -inf), so a tensor is
 *     accepted or refused the same way by both calls: sticky JSS_FLAG_ERROR, env unchanged, JSS_ACTION_SKIP, log_prob
 *     NaN.  The test comes before the coin: whether an env errors never depends on the RNG, also at epsilon = 1.
 *   Greedy action g: the legal action with the largest score, ties to the lowest index, the scores compared as IEEE
 *     floats (-0.0 and +0.0 tie): np.argmax / torch.argmax over the legal entries.
 *   Exploration: with H = jss_hash_env, h_env = jss_hash3 of (seed, env_id_base + i, step_index) (jss_rng.h) and
 *     T = floor(epsilon * 2^32) (computed in double, exact, 0 <= T <= 2^32), the env explores iff H(h_env, 0) < T, and
 *     then takes the action jss_pick maps (H(h_env, 1), n) to, over the set bits of its action_mask in ascending order,
 *     n the number of legal actions (a legal no-op included): the mapping of JSS_RULE_RANDOM.  The coin and the pick use separate
 *     hashes, so a small epsilon does not favour the lowest legal actions.  With epsilon = 0 the result does not depend
 *     on seed or step_index.
 *   log_prob_out_dev[i] = log((a == g ? 1 - e : 0) + e / n), e = T * 2^-32, in fp32: the log-probability of a under
 *     the epsilon-greedy policy that chose it; exactly 0.0 whenever epsilon = 0.
 *   Special cases: those of jss_step_logits() (done env: action 0, log_prob 0; only the no-op legal: action J_i,
 *     log_prob 0, its score not read; no legal action at all: JSS_ACTION_SKIP, NaN).
 *   actions_out_dev: device int32[N] (required); log_prob_out_dev: device fp32[N], NULL skips that store.
 *   Returns JSS_ERR_INVALID for a NULL scores_dev / actions_out_dev, ld < jobs_max + 1, or epsilon NaN or outside
 *   [0, 1].
 * Bytes per ta80 env-step: 5 604, those of jss_step_logits().  Measured on an H100 SXM 80 GB HBM3 at a 700 W power
 * limit (ta80, N = 65 536, median of three runs): 155.8 us per step at epsilon = 0 and 156.3 us at 0.05, against
 * 260.5 us for masked_fill + argmax + jss_step() in torch and 159.9 us for jss_step_logits() (DESIGN.md section 4). */
int jss_step_greedy(jss_t *h, const float *scores_dev, int64_t ld, double epsilon, uint64_t seed, uint64_t step_index,
                    int32_t *actions_out_dev, float *log_prob_out_dev, void *stream);

/* jss_step_greedy() that records the transition into the caller's rollout slot: it is to jss_step_greedy() what
 * jss_step_logits_record() is to jss_step_logits().  The same slot layouts, 16-byte alignment rule (JSS_ERR_INVALID
 * for a NULL or misaligned slot pointer) and zero-reward record of an unchanged env; real_obs is left stale
 * (jss_refresh_obs()). */
int jss_step_greedy_record(jss_t *h, const float *scores_dev, int64_t ld, double epsilon, uint64_t seed,
                           uint64_t step_index, int32_t *actions_out_dev, float *log_prob_out_dev, float *obs_out_dev,
                           uint8_t *mask_out_dev, int32_t *scalars_out_dev, void *stream);

/* Rewrite real_obs from the state blocks after jss_step_logits_record(); returns at once when nothing is stale. */
int jss_refresh_obs(jss_t *h, void *stream);

/* Replaces DispatchingRule.run_episode (dispatching.py:55-75) for the whole
 * batch: n_steps x (policy -> step) fused in one launch, state kept on chip
 * between steps; observations are written every step iff write_obs != 0. */
int jss_rollout(jss_t *h, int rule, uint64_t seed, uint64_t step_index, int n_steps,
                int write_obs, void *stream);

/* jss_rollout() that also RECORDS the trajectory (what an on-policy collector wants from a rule / random policy):
 * for k < n_steps and env e, slot k * N + e of the caller's device buffers receives the outputs of transition k --
 * traj_obs [n_steps][N][J][7] fp32, traj_mask [n_steps][N][mask_stride] u8, traj_scalars [n_steps][N][4] int32
 * (the 16-byte records), traj_actions [n_steps][N] int32 (the action taken; may be NULL).  The regular buffers hold
 * the last transition afterwards, as after jss_rollout.  n_steps * N < 2^31. */
int jss_rollout_traj(jss_t *h, int rule, uint64_t seed, uint64_t step_index, int n_steps, float *traj_obs,
                     uint8_t *traj_mask, int32_t *traj_scalars, int32_t *traj_actions, void *stream);

/* Runs a caller's static priority rule (DispatchingRule.run_episode, dispatching.py:21-75, with a table for the
 * rule's key) to the end of every env's episode in one launch per lane class present: random-key / evolutionary
 * metaheuristics scoring candidate priorities by makespan, one-shot priority policies, custom static rules.
 *   Table: env i's priority of operation k of job j is prio_dev[i*ld_env + j*ld_job + k*ld_op] (device fp32), read
 *     only for j < J_i and k < M_i.  Strides are in elements, may be 0 (broadcast) and are used in 64-bit index
 *     arithmetic.  Only the entry of a legal job's current operation (k = todo_time_step_job[j]) is ever read.
 *   Decision: among the legal jobs, the one with the largest priority; ties to the lowest job index; priorities are
 *     compared as IEEE floats, so -0.0 and +0.0 tie (the argmax of jss_step_greedy()).  The no-op is taken only when no
 *     job is legal and the no-op is (what the built-in rules do under JSS_COIN_NEVER).  There is no RNG: the result
 *     does not depend on seed or step index.
 *   Bad priorities (a NaN or +inf on a legal job's current operation, or every legal job at -inf: the bad-row rule of
 *     jss_step_greedy()): the env gets the sticky JSS_FLAG_ERROR bit, is left in its state before that decision and
 *     gets no further decisions in this call.
 *   Loop: each env makes at most n_steps decisions and stops at the end of its episode.  An env never resets inside
 *     the call, also under JSS_CREATE_AUTO_RESET, and an env that is done when the call starts is left untouched
 *     (unlike jss_rollout(): the same table would only replay the same episode).  Episode statistics, solution
 *     (JSS_CREATE_RECORD_SOLUTION) and jss_stats() are updated as by jss_step().  Afterwards every env's buffers
 *     (real_obs, action_mask, the scalar record with the last transition's reward) hold its final state, as after
 *     jss_rollout(write_obs = 0): an env equals a twin stepped with jss_step_greedy(rows, epsilon = 0) up to n_steps
 *     times, rows[j] = the priority of job j's current operation and the no-op column -inf.
 *   n_steps = 0 does nothing.  Returns JSS_ERR_INVALID for a NULL or not 4-byte-aligned prio_dev, a negative stride or
 *     n_steps < 0, and JSS_ERR_STATE before jss_assign().
 * Bytes per ta80 decision: the 4-byte priority of each legal job's current operation (L2 / HBM), nothing else; the
 * state block is read and written once per call and the outputs written once.  Measured on an H100 SXM 80 GB HBM3 at
 * a 700 W power limit (ta80, N = 65 536, reset to done, 2 000 decisions per episode, median of three rounds): 119.9 ms
 * per batch with per-operation priorities (1.09 G decisions/s), against 1 259.8 ms for export_state + a torch gather
 * + jss_step_greedy per decision; 118.1 ms with per-job priorities against 332.8 ms for the jss_step_greedy loop on
 * the static row (DESIGN.md section 4). */
int jss_rollout_priority(jss_t *h, const float *prio_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op, int n_steps,
                         void *stream);

/* jss_rollout_priority() with every decision drawn from a softmax over a caller's logit table instead of its argmax,
 * and each episode's log-probability and its gradient with respect to the table: sampling decoding of a one-shot
 * scoring network (many schedules per instance from one broadcast table), ant-colony / cross-entropy search, and
 * policy-gradient training of a network that emits per-operation logits once per instance.
 *   Table, loop, done envs, outputs, n_steps = 0 and launches: those of jss_rollout_priority(), logits_dev in place of
 *     prio_dev.  Only the entry of a legal job's current operation is ever read.
 *   Decision d (0-based, counted per env within the call, no-op decisions included) of env i: with
 *     h = jss_hash3(seed, env_id_base + i, step_index + d) and x_j the entry of job j's current operation, the
 *     Gumbel-max draw of jss_step_logits() over the legal jobs, a = argmax((x_j - mx) + g_j) in fp32 with mx the
 *     largest legal x_j and g_j the Gumbel noise that call draws for action j from h, ties to the lowest index, with
 *     log-probability (x_a - mx) - log sum exp(x - mx) over the legal jobs.  Like jss_step_logits(), it can draw
 *     differently for a given seed than builds that keyed on x_j + g_j, where the fp32 rounding of that sum decided.
 *     It equals, bit for bit, jss_step_logits(rows, seed, step_index + d) on the row rows[j] = x_j, no-op column -inf.
 *     The no-op is taken only when no job is legal and it is; that decision draws nothing and has log-probability 0.
 *   Bad entries (a NaN or +inf on a legal job's current operation, or every legal job at -inf: the bad-row rule of
 *     jss_step_logits()): the env gets the sticky JSS_FLAG_ERROR bit, is left in its state before that decision and
 *     gets no further decisions in this call.
 *   log_prob_out_dev (device fp32 [N], required): env i's sum of its decisions' log-probabilities in this call, added
 *     in fp32 in decision order; 0 for an env that is done at entry or makes no decision; NaN for an env a decision of
 *     this call leaves with the error bit.
 *   grad_out_dev (device fp32 [N][jobs_max][machines_max], contiguous: the layout of solution; NULL: no gradient):
 *     G[i][j][k] = d log_prob_out[i] / d (env i's entry of operation k of job j)
 *                = sum over env i's decisions t of (1[job j drawn at t] - p_t(j)) * 1[j legal at t and todo_j = k],
 *     p_t the softmax over the legal jobs at t.  Every entry j < J_i, k < M_i is written, 0 for operations finished
 *     before the call or never reached and for an env done at entry; an env that gets NaN gets all-zero rows, so that
 *     masking it out leaves no NaN in a backward pass.  Entries past J_i / M_i are not written.  The kernel adds each
 *     job's p_t in a register while its operation is current and stores the entry once, when the job is drawn: one
 *     4-byte store per decision, the table of gradients is never read.
 *   Returns JSS_ERR_INVALID for a NULL or not 4-byte-aligned logits_dev or log_prob_out_dev, a misaligned grad_out_dev,
 *     a negative stride or n_steps < 0, and JSS_ERR_STATE before jss_assign().
 * Measured on an H100 SXM 80 GB HBM3 at a 400 W power limit (ta80, N = 65 536, reset to done, 2 000 decisions per
 * episode, median of three rounds): 156.6 ms per batch without the gradient, 162.2 ms with it and the torch backward,
 * against 120.7 ms for jss_rollout_priority() on the same table and 1 330.1 ms for export_state + a torch gather +
 * jss_step_logits per decision (DESIGN.md section 4). */
int jss_rollout_priority_sample(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                                uint64_t seed, uint64_t step_index, int n_steps, float *log_prob_out_dev,
                                float *grad_out_dev, void *stream);

/* jss_rollout_priority_sample() with each episode's policy entropy, the regulariser of REINFORCE and PPO on a table
 * policy, and its gradient.  Every draw, state, log_prob_out and grad_out entry, RNG counter advance and error bit is
 * bit for bit what jss_rollout_priority_sample() gives with the same arguments.
 *   Entropy of a decision with legal jobs L: with x_j, mx, d_j = x_j - mx, e_j = exp(d_j) and S = sum_{j in L} e_j the
 *     values the draw computes (fast exp / log), H_t = log S - T / S, T = sum over j in L with e_j > 0 of e_j d_j,
 *     summed in S's order.  A term with e_j = 0 adds nothing (no 0 * -inf), and a decision with one job of nonzero
 *     probability gives exactly +0.
 *   entropy_out_dev (device fp32 [N], required): env i's fp32 sum of H_t over its decisions of this call, in decision
 *     order; forced no-ops add 0; 0 for an env done at entry or making no decision; NaN wherever log_prob_out is NaN.
 *   entropy_grad_out_dev (device fp32 [N][jobs_max][machines_max], the layout of grad_out; NULL: none):
 *     d entropy_out[i] / d (entry of operation k of job j) = sum over the decisions t where j is legal at operation k
 *     of -p_t(j) (lp_t(j) + H_t), p = e_j / S and lp = d_j - log S (0 where p = 0).  Written where grad_out is, with
 *     grad_out's zeros: operations finished before the call or never reached, envs done at entry, all-zero rows for an
 *     env that gets NaN.  Either gradient pointer may be NULL.
 *   Returns the errors of jss_rollout_priority_sample(), and JSS_ERR_INVALID for a NULL or not 4-byte-aligned
 *     entropy_out_dev or a misaligned entropy_grad_out_dev. */
int jss_rollout_priority_sample_entropy(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job,
                                        int64_t ld_op, uint64_t seed, uint64_t step_index, int n_steps,
                                        float *log_prob_out_dev, float *entropy_out_dev, float *grad_out_dev,
                                        float *entropy_grad_out_dev, void *stream);

/* Values every legal action of every env by a dispatching-rule rollout to the end of its episode, in one launch per
 * lane class present, and changes nothing but the caller's table: the reference's copy.deepcopy(env) + step(a) +
 * DispatchingRule.run_episode (dispatching.py:55-75) per legal action.  For the rollout (pilot) method -- take the
 * action with the smallest value, repeat; with a deterministic rule never worse than the rule alone -- per-action
 * teacher labels for imitation learning, and leaf values for tree search.
 *   Candidates: the legal actions of env i's current state, the set bits of its action_mask row (jobs 0..J_i-1 and
 *     the no-op J_i when it is legal).
 *   Value: makespan_out_dev[i*ld + a] (device int32, 64-bit index arithmetic) is the current_time_step at which env
 *     i's episode ends if it takes a now and then follows rule to the end.  The rule (any JSS_RULE_*, RANDOM
 *     included) decides as jss_policy(rule, coin_mode, ...) would: its decision d (0-based, counted after the
 *     candidate's step) hashes h = jss_hash3(seed, env_id_base + i, step_index + d), so every candidate of an env sees
 *     the same random numbers, and CR uses the handle's due-date factor (jss_set_cr_due_date_factor()).  Equivalently,
 *     a twin batch (same instances and env_id_base, auto-reset off, env i in the same state) stepped with a and then
 *     with jss_policy(rule, coin_mode, seed, step_index + d) + jss_step() for d = 0, 1, ... until done ends at
 *     current_time_step == makespan_out[i][a]; under JSS_COIN_DEVICE that tail is jss_rollout(rule, seed,
 *     step_index, n).  Each candidate gets at most 2*J_i*M_i + 1 rule decisions (no episode is longer).
 *   -1 is written for every column 0..J_i that is not a legal action, every column 0..J_i of an env that is done at
 *     entry, and a candidate whose rollout stops before done: the rule finds nothing legal, a step leaves the env
 *     unchanged with the error bit, or the bound trips (none of which a state reached from jss_reset() leads to).
 *     Columns J_i+1 .. ld-1 are not written.
 *   No side effects: state blocks, real_obs, action_mask, the scalar records, solution, episode statistics,
 *     jss_stats(), flags and the stale-real_obs marker are as before, under JSS_CREATE_AUTO_RESET and
 *     JSS_CREATE_RECORD_SOLUTION too.  An env with the sticky error bit is valued like any other.  The call reads only
 *     the state blocks and neither needs nor triggers jss_refresh_obs().
 *   Returns JSS_ERR_INVALID for a bad rule or coin mode, a NULL or not 4-byte-aligned makespan_out_dev or
 *     ld < jobs_max + 1, and JSS_ERR_STATE before jss_assign().
 * Bytes: per candidate the env's state block (L2) and one 4-byte store; per rule decision nothing beyond the staged
 * instance tables.  One warp simulates one (env, candidate) at a time; a batch too small to fill the SMs spreads each
 * env's candidates over several warps.  Measured on an H100 SXM 80 GB HBM3 at a 700 W power limit (MWR, device coin,
 * median of three rounds): ta80 at N = 4 096 from reset 888.2 ms per call (409 600 candidates, 947 M decisions/s)
 * against 1 969.5 ms for import_state + jss_step + jss_rollout per candidate column; after 500 random decisions 96.5
 * against 1 631.3 ms; ta80 at N = 32 8.9 against 496.9 ms; ta01 at N = 65 536 101.3 against 185.0 ms (DESIGN.md
 * section 4). */
int jss_lookahead(jss_t *h, int rule, int coin_mode, uint64_t seed, uint64_t step_index, int32_t *makespan_out_dev,
                  int64_t ld, void *stream);

/* jss_lookahead() with the greedy decisions of a caller's priority table in place of a dispatching rule: every legal
 * action of every env valued by a rollout of the table to the end of its episode, in one launch per lane class present,
 * changing nothing but the caller's values.  The rollout method improves any deterministic base policy: the argmin of
 * these values, taken at every decision, is never worse than the table's own greedy decode (jss_rollout_priority()),
 * and it is the imitation label of expert iteration for the network that emitted the table.
 *   Table: that of jss_rollout_priority(), entry prio_dev[i*ld_env + j*ld_job + k*ld_op] (strides in elements, 0 to
 *     broadcast, 64-bit index arithmetic).  Only the entry of a legal job's current operation is ever read.
 *   Candidates: those of jss_lookahead(), the set bits of env i's action_mask row.  The candidate is taken whatever its
 *     priority, the no-op included (which the table's own decisions take only when no job is legal).
 *   Value: makespan_out_dev[i*ld + a] is the current_time_step at which env i's episode ends if it takes a now and then
 *     follows the table's decision of jss_rollout_priority(): the legal job whose current operation has the largest
 *     priority, ties to the lowest index under IEEE comparison (-0.0 and +0.0 tie), the no-op only when no job is
 *     legal.  Equivalently, a twin batch (same instances and env_id_base, auto-reset off, env i in the same state)
 *     stepped with a and then with jss_rollout_priority(table, 2*J*M + 1) ends done at current_time_step ==
 *     makespan_out[i][a].  Each candidate gets at most 2*J_i*M_i + 1 table decisions.  No RNG: the values depend on
 *     neither seed nor step counter.
 *   -1 is written as by jss_lookahead() (illegal columns 0..J_i, every column 0..J_i of an env done at entry), and for
 *     a candidate whose rollout stops before done: a bad table at one of its decisions (a NaN or +inf on a legal job's
 *     current operation, or every legal job at -inf: the bad-row rule of jss_rollout_priority()), nothing legal, a
 *     step that leaves the env unchanged with the error bit, or the bound.  A bad table costs only the candidates whose
 *     rollouts meet it and sets no error bit anywhere.  Columns J_i+1 .. ld-1 are not written.
 *   No side effects: those of jss_lookahead().  The call reads only the state blocks and neither needs nor triggers
 *     jss_refresh_obs().
 *   Returns JSS_ERR_INVALID for a NULL or not 4-byte-aligned prio_dev or makespan_out_dev, a negative stride or
 *     ld < jobs_max + 1, and JSS_ERR_STATE before jss_assign().
 * Bytes: those of jss_lookahead(), plus per table decision the 4-byte priority of each legal job's current operation
 * (L2 / HBM) in place of the suffix sums in shared memory.  Measured on an H100 SXM 80 GB HBM3 at a 700 W power limit
 * (seeded per-env (N, J, M) table, median of three rounds): ta80 at N = 4 096 from reset 644.3 ms per call (409 600
 * candidates, 1.27 G decisions/s) against 953.0 ms for import_state + jss_step + jss_rollout_priority per candidate
 * column; after 500 random decisions 58.9 against 752.4 ms; ta80 at N = 32 6.64 against 347.4 ms; ta01 at N = 65 536
 * 85.1 against 119.5 ms.  The MWR table runs 13-41 % faster than jss_lookahead(MWR, JSS_COIN_NEVER) on the same values
 * (DESIGN.md section 4). */
int jss_lookahead_priority(jss_t *h, const float *prio_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                           int32_t *makespan_out_dev, int64_t ld, void *stream);

/* k episodes per env drawn from a caller's logit table, in one launch per lane class present, leaving the envs
 * untouched: the several sampled episodes from one state that a shared-baseline (POMO-style, self-critical) REINFORCE
 * loss and a best-of-k sampling decode need, without a batch of N*k envs or N*k copies of the table.
 *   Table: that of jss_rollout_priority_sample(), entry logits_dev[i*ld_env + j*ld_job + k*ld_op].
 *   Sample s = 0 .. k-1 of env i: with B = 2*J*M + 1 (J and M the batch maxima, the default n_steps of
 *     jss_rollout_priority_sample()), at most B decisions from env i's current state, decision d at RNG counter
 *     step_index + s*B + d and otherwise exactly jss_rollout_priority_sample()'s decision (hash, Gumbel-max draw,
 *     log-probability, bad-table rule).  Equivalently: a twin batch (same instances and env_id_base, auto-reset off, env
 *     i in the same state) run once with jss_rollout_priority_sample(logits, seed, step_index + s*B, B).
 *   Outputs (device, row stride ld, 64-bit index arithmetic): makespan_out_dev[i*ld + s] (int32) is the twin's
 *     current_time_step if it ends done, else -1; log_prob_out_dev[i*ld + s] (fp32) is the twin's log_prob, bit for
 *     bit, NaN where a decision meets a bad table.  An env done at entry gets -1 and 0 in every column.  Columns k ..
 *     ld-1 are not written.  How each env's samples are spread over work items is the library's choice and changes no
 *     output.
 *   No side effects: those of jss_lookahead(), and no error bit is set.  The call reads only the state blocks and
 *     neither needs nor triggers jss_refresh_obs().
 *   Returns JSS_ERR_INVALID for a NULL or not 4-byte-aligned pointer, a negative stride, k < 1, ld < k or k*B past
 *     2^64, JSS_ERR_UNSUPPORTED for k >= 2^31, and JSS_ERR_STATE before jss_assign().
 * Measured on an H100 SXM 80 GB HBM3 at a 700 W power limit (seeded tables, median of three rounds): ta80 at N = 256,
 * k = 64 after 500 random decisions 29.8 ms per call against 241.4 ms for import_state + jss_rollout_priority_sample
 * per sample; ta80 at N = 1, k = 4 096 from reset 24.6 ms against 9.9 ms for a 4 096-env batch, whose memory the call
 * does not need (DESIGN.md section 4). */
int jss_sample_episodes(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                        uint64_t seed, uint64_t step_index, int64_t k, int32_t *makespan_out_dev,
                        float *log_prob_out_dev, int64_t ld, void *stream);

/* The backward of jss_sample_episodes() with the same table, seed, step_index and k, from the same state: it replays
 * the draws and adds sum_s weights[i*ld + s] * G_s[i] into grad_out_dev (device fp32
 * [split][N][jobs_max][machines_max], zero-filled by the caller).  G_s[i] is what jss_rollout_priority_sample()'s
 * grad_out holds for the twin of sample s: zero for a sample with log-probability NaN and for an env done at entry.
 * Chunk c takes the samples s = c, c + split, ... in increasing s; each entry is read and written by the one lane that
 * owns its job, with no atomics, so the result is deterministic for a given split.  The caller sums over c; a split > 1
 * lets a small N fill the GPU while the partial buffer stays split*N*J*M floats.  Samples of weight 0 cost nothing.
 * Returns the errors of jss_sample_episodes() (weights_dev and grad_out_dev in place of its outputs) and
 * JSS_ERR_INVALID for split < 1 or split > k. */
int jss_sample_episodes_grad(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                             uint64_t seed, uint64_t step_index, int64_t k, const float *weights_dev, int64_t ld,
                             int split, float *grad_out_dev, void *stream);

/* jss_sample_episodes() with each sample's policy entropy: entropy_out_dev[i*ld + s] (device fp32) is what
 * jss_rollout_priority_sample_entropy() reports for the twin of sample s, bit for bit; 0 for an env done at entry.
 * makespan_out_dev and log_prob_out_dev are bit for bit jss_sample_episodes()'s.  Returns the errors of
 * jss_sample_episodes(), entropy_out_dev checked as its outputs are. */
int jss_sample_episodes_entropy(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                                uint64_t seed, uint64_t step_index, int64_t k, int32_t *makespan_out_dev,
                                float *log_prob_out_dev, float *entropy_out_dev, int64_t ld, void *stream);

/* The backward of jss_sample_episodes_entropy(): one replay of the draws that adds sum_s (weights[i*ld + s] * G_s[i] +
 * entropy_weights[i*ld + s] * GH_s[i]) into grad_out_dev, G_s and GH_s the grad_out and entropy_grad_out of
 * jss_rollout_priority_sample_entropy() for the twin of sample s.  Chunking, ownership and determinism are those of
 * jss_sample_episodes_grad(); a sample adds w G first, so entropy weights of 0 add what jss_sample_episodes_grad()
 * adds, bit for bit.  Samples with both weights 0 cost nothing.  Returns the errors of jss_sample_episodes_grad(),
 * entropy_weights_dev checked as weights_dev is. */
int jss_sample_episodes_entropy_grad(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                                     uint64_t seed, uint64_t step_index, int64_t k, const float *weights_dev,
                                     const float *entropy_weights_dev, int64_t ld, int split, float *grad_out_dev,
                                     void *stream);

/* The schedule of one sample per env of jss_sample_episodes() (same table, seed and step_index, same state): env i
 * replays sample sample_dev[i] (device int32 [N]; < 0 skips the env) and writes the start time of every operation that
 * sample starts into solution_out_dev[i][j][k] (device int32 [N][jobs_max][machines_max], the layout of solution).
 * Every other entry is left alone.  Returns the table errors of jss_sample_episodes(), JSS_ERR_INVALID for a NULL or
 * not 4-byte-aligned sample_dev or solution_out_dev, and JSS_ERR_STATE before jss_assign(). */
int jss_sample_episodes_solution(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                                 uint64_t seed, uint64_t step_index, const int32_t *sample_dev,
                                 int32_t *solution_out_dev, void *stream);

/* jss_lookahead() with k episodes drawn from a caller's logit table after each candidate: every legal action of every
 * env valued by k sampled rollouts to the end of its episode, in one launch per lane class present, changing nothing
 * but the caller's values.  These are the action values Q(s, a) of the table's stochastic policy that a rollout
 * policy-improvement step (argmin of the mean or best-of-k), a soft improvement target exp(-Q / tau) or a per-action
 * baseline needs, without a twin batch and an import, a step and a jss_sample_episodes() per candidate.
 *   Table: that of jss_rollout_priority_sample(), entry logits_dev[i*ld_env + j*ld_job + k*ld_op].
 *   Candidates: those of jss_lookahead(), the set bits of env i's action_mask row, each taken whatever its logit.
 *   Value: with B = 2*J*M + 1 (J and M the batch maxima, the B of jss_sample_episodes()), makespan_out_dev[i*ld + a*k +
 *     s] is the current_time_step at which env i's episode ends if it takes a now and then draws at most B decisions,
 *     decision d at RNG counter step_index + s*B + d, exactly as sample s of jss_sample_episodes() draws them.
 *     Equivalently: a twin batch (same instances, seed and env_id_base, auto-reset off, env i in the same state)
 *     stepped with a and then run with jss_sample_episodes(logits, seed, step_index, k) has column s of its makespan
 *     equal to makespan_out[i][a*k + s]; where the step alone ends the episode, every s holds that end time.  Common
 *     random numbers: every candidate of an env uses the same counters, so differences between candidates reflect the
 *     action, not the noise.
 *   -1 is written for every pair of an illegal column 0..J_i, every pair of an env done at entry, a candidate step that
 *     leaves the env unchanged with the error bit, and a sample that stops before done: nothing legal, a bad table at
 *     one of its decisions (the bad-row rule of jss_rollout_priority_sample(); no error bit is set), or the bound.
 *     Entries (J_i+1)*k .. ld-1 are not written.  How each env's pairs are spread over work items is the library's
 *     choice and changes no output.
 *   No side effects: those of jss_lookahead().  The call reads only the state blocks and neither needs nor triggers
 *     jss_refresh_obs().
 *   Returns JSS_ERR_INVALID for a NULL or not 4-byte-aligned pointer, a negative stride, k < 1, k*B past 2^64 or
 *     ld < (jobs_max + 1)*k, JSS_ERR_UNSUPPORTED for k >= 2^31 or tiles*(jobs_max + 1)*k >= 2^31 (tiles: at most one
 *     per 8 envs of an instance), and JSS_ERR_STATE before jss_assign().
 * Cost: about one jss_sample_episodes() sample per (legal candidate, s) pair.  Measured on an H100 SXM 80 GB HBM3 at a
 * 700 W power limit (seeded per-env table, median of three rounds): ta80 at N = 256, k = 16 from reset 831.8 ms per
 * call against 889.8 ms for import_state + jss_step + jss_sample_episodes per candidate column; after 500 random
 * decisions 83.0 against 701.4 ms; ta01 at N = 4 096, k = 8 53.9 against 68.6 ms (DESIGN.md section 4). */
int jss_lookahead_sample(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                         uint64_t seed, uint64_t step_index, int64_t k, int32_t *makespan_out_dev, int64_t ld,
                         void *stream);

/* Beam search over a caller's logit table, in one launch per lane class present, leaving the envs untouched: the W
 * most likely schedules per env under the table's softmax policy, keeping W partial schedules per env on chip (one CTA
 * per env, the beams' state blocks in shared memory).  Deterministic: no RNG, no seed.
 *   Table: that of jss_rollout_priority_sample(), entry logits_dev[i*ld_env + j*ld_job + k*ld_op] (strides in
 *     elements, 0 to broadcast, 64-bit index arithmetic).  Only the entry of a legal job's current operation is read.
 *   Rounds: a round allocates exactly one job.  Env i starts from its current state with one beam (slot 0, score +0.0)
 *     and runs R_i = sum_j (M_i - todo_j - [tufco_j > 0]) rounds, the operations not yet started at entry: every beam
 *     allocates one per round, so all complete beams finish together.  At the start of a round a beam with no legal job
 *     but a legal no-op takes the no-op (log-probability 0), as long as that holds; the search takes no other no-op.
 *   Children: the candidates of a beam are its legal jobs j, with score + logp_j added in fp32, logp_j = (x_j - mx) -
 *     log(sum exp(x - mx)) over the legal jobs computed as jss_rollout_priority_sample() computes the log-probability of
 *     the job it draws (same reductions, same fast exp / log).  So a slot's score is, bit for bit, the log_prob that
 *     jss_rollout_priority_sample() reports for an episode drawing the same jobs from the same state.  A job with
 *     logp_j = -inf is not a candidate.  A beam whose decision meets a bad row (NaN or +inf on a legal job's current
 *     operation, or every legal job at -inf) is dropped, as is a beam with nothing legal (an imported state).
 *   Selection: the W best candidates of all beams under one total order -- score descending (IEEE compare, -0 and +0
 *     tie), then parent slot ascending, then job ascending -- become slots 0 .. W-1 in that order.  Equal states are
 *     not merged.  The result does not depend on the grid, the batch order or sharding.
 *   Outputs (device, row stride ld >= width): makespan_out_dev[i*ld + b] (int32) and score_out_dev[i*ld + b] (fp32)
 *     of final slot b: its end time and score; -1 and -inf for a slot without a complete beam; -1 and NaN in every slot
 *     of an env that ends with no complete beam after dropping one for a bad row; -1 and 0 in every slot of an env done
 *     at entry.  Columns width .. ld-1 are not written.
 *   order_out_dev (NULL, or device int32 [N][jobs_max][machines_max], the layout of solution): order_out[i][j][k] is the
 *     round at which the best slot (smallest makespan, ties to the lowest slot) allocates operation k of job j; -1 for
 *     the operations started before the call and in every entry of an env without a complete beam.  Entries past
 *     J_i / M_i are not written.  jss_rollout_priority() on the table -order from the same state replays that beam and
 *     ends done at makespan_out[i*ld + best]: its next job always holds the largest -round among the legal jobs.
 *   No side effects: those of jss_lookahead(); no error bit is set and the RNG counter does not move.  An env with the
 *     sticky error bit is searched like any other.  The call neither needs nor triggers jss_refresh_obs().
 *   Memory: 2*W state blocks per CTA in shared memory (72 KB for ta80 at W = 32, 177 KB for 256 x 32), and, with
 *     order_out_dev, a per-round backpointer trace owned by the handle (2 bytes per slot and round for each resident
 *     CTA: about 17 MB for ta80 at W = 16 on 132 SMs), allocated by the first call that needs it and freed by
 *     jss_destroy().  Calls with order_out_dev on one handle share that trace: do not let them overlap on different
 *     streams.
 *   Returns JSS_ERR_INVALID for a NULL (order_out_dev aside) or not 4-byte-aligned pointer, a negative stride, width <
 *     1 or > JSS_MAX_BEAM_WIDTH, or ld < width; JSS_ERR_CUDA if the trace cannot be allocated; JSS_ERR_STATE before
 *     jss_assign().
 * Measured on an H100 SXM 80 GB HBM3 at a 700 W power limit (seeded per-env tables, median of three rounds): ta80 at
 * N = 256, W = 16 from reset 30.1 ms per call (272 M beam decisions/s) against 2 232 ms for the torch loop of
 * export_state / top-W / import_state / jss_step on N*W envs; after 500 random decisions 23.3 against 1 879 ms; ta01 at
 * N = 4 096, W = 8 8.86 against 324 ms (DESIGN.md section 4). */
int jss_beam_search(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op, int width,
                    int32_t *makespan_out_dev, float *score_out_dev, int64_t ld, int32_t *order_out_dev, void *stream);

/* Stochastic beam search (Kool, van Hoof, Welling, ICML 2019) over a caller's logit table, in one launch per lane class
 * present, leaving the envs untouched: W *distinct* episodes per env drawn without replacement from the distribution
 * jss_rollout_priority_sample() samples from, each with its perturbed log-probability (its key).
 *   Shared with jss_beam_search(): the table, the rounds, forced no-ops, the candidates (legal jobs with logp_j > -inf),
 *     the dropping of beams on bad rows, done-at-entry envs and 1 <= W <= JSS_MAX_BEAM_WIDTH.  A slot's log_prob is its
 *     beam score, accumulated as jss_beam_search() accumulates it, so it equals, bit for bit, the log_prob
 *     jss_rollout_priority_sample() reports for the same episode.
 *   Perturbation (top-down Gumbel): the root beam has key T = 0.  In round r a beam in slot b with score phi_b and key
 *     T_b gives each candidate j the value G_j = (phi_b + lp_j) + g_j, g_j = -log(-log u), u = ((H(h, b * 256 + j) >> 8)
 *     + 0.5) * 2^-24, H = jss_hash_env and h = jss_hash3(seed, env_id_base + i, step_index + r) (jss_rng.h): the
 *     uniforms can be restated on the host.  With Z = max_j G_j, the candidate
 *     attaining Z (lowest job on ties) gets key exactly T_b, every other one min(T_b, T_b - max(v, 0) - log1p(e^-|v|)),
 *     v = T_b - G_j + log(1 - e^(G_j - Z)).
 *   Selection: that of jss_beam_search() with the key in place of the score (key descending, then parent slot, then
 *     job); the W best become slots 0 .. W-1.
 *   Outputs (device, row stride ld >= width): makespan_out_dev[i*ld + b] (int32), log_prob_out_dev and key_out_dev
 *     (fp32) of final slot b; -1 / -inf / -inf for a slot without a complete beam; -1 / NaN / NaN in every slot of an env
 *     whose beams all met a bad row; -1 / 0 / 0 in every slot of an env done at entry.  Columns width .. ld-1 are not
 *     written.
 *   order_out_dev (NULL, or device int32 [N][width][jobs_max][machines_max]): every slot's allocation round of each
 *     operation, in jss_beam_search()'s order format; -1 for operations started before the call and in every entry of a
 *     slot without a complete beam.  Entries past J_i / M_i are not written.  It uses jss_beam_search()'s handle-owned
 *     trace under the same rule: calls with an order on one handle must not overlap on different streams.
 *   No side effects, as jss_beam_search(); the call reads the RNG counters step_index .. step_index + R_i - 1.
 *   Returns JSS_ERR_INVALID for a NULL (order_out_dev aside) or not 4-byte-aligned pointer, a negative stride, width < 1
 *     or > JSS_MAX_BEAM_WIDTH, or ld < width; JSS_ERR_CUDA if the trace cannot be allocated; JSS_ERR_STATE before
 *     jss_assign(). */
int jss_sample_without_replacement(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                                   uint64_t seed, uint64_t step_index, int width, int32_t *makespan_out_dev,
                                   float *log_prob_out_dev, float *key_out_dev, int64_t ld, int32_t *order_out_dev,
                                   void *stream);

/* One round of beam search for a policy that reads the observation at every decision: the per-round form of
 * jss_beam_search(), with a logit row per beam in place of the table, on a handle whose envs are the beams.  One launch
 * per lane class present (one group per CTA).
 *   Groups: the N envs form G = N / width groups; group g is envs g*W .. g*W + W-1 and its slot b is env g*W + b.  Every
 *     env of a group must run the same instance: a group is one search.
 *   Scores: score_dev, caller-owned fp32 [N], is read and written.  A slot is live iff its score is finite.  A search
 *     starts with score = [0, -inf, ..., -inf] per group and its start state in slot 0; the other slots' states are
 *     never read.
 *   Rows: logits_dev[env*ld + j] (ld >= jobs_max + 1), read only at the legal jobs j of a live, not-done beam; the no-op
 *     column is never read.
 *   One call is one round of jss_beam_search() per group, so that rows gathered from a table at each slot's todo give
 *     jss_beam_search()'s result bit for bit:
 *     1. Expand: a live, not-done beam with a legal job has as candidates its legal jobs j with score + logp_j > -inf,
 *        logp_j computed as jss_beam_search() computes it with x_j = row[j].  A bad row (NaN or +inf at a legal job, or
 *        every legal job at -inf) gives no candidate and sets the group's bad_out; a live beam with no legal job, or
 *        done, gives none.
 *     2. Select: the W best candidates in jss_beam_search()'s order (score descending, -0 = +0, then parent slot, then
 *        job) become slots 0 .. nn-1.
 *     3. Step: new slot b gets its parent's state as at call entry, stepped with its job, then the no-op as long as no
 *        job is legal and the no-op is.  Its score is the candidate's, or NaN if a step fails (an imported state).
 *        Slots nn .. W-1 get score -inf; their state is left as it is (stale).
 *     A group without a live, not-done beam is untouched: its states and scores are left as they are.
 *   Outputs (device int32): parent_out_dev[env] and action_out_dev[env], the new slot's parent slot and job, -1 / -1 for
 *     an empty slot, b / -1 for slot b of an untouched group (so a walk back through the rounds is uniform);
 *     bad_out_dev[g] is 1 if a beam of group g met a bad row in this call, else 0.
 *   A written slot's state block, real_obs row, action_mask row and scalar record equal, bit for bit, those of a twin
 *     that ran jss_step(job) and then jss_step(J) for each forced no-op; the rows are written whole.  Statistics,
 *     solution, the error bit and auto-reset are not touched, and no RNG is used.  A stale real_obs is refreshed first.
 *   Returns JSS_ERR_INVALID for a NULL or not 4-byte-aligned pointer, width < 1 or > JSS_MAX_BEAM_WIDTH, N not divisible
 *     by width, ld < jobs_max + 1 or a group that mixes instances; JSS_ERR_STATE before jss_assign().
 * Measured on an H100 SXM 80 GB HBM3 at a 700 W power limit with a linear policy on real_obs in torch (median of three
 * rounds): ta80 at G = 256, W = 16 from reset 288 ms per search (144 us per round, policy included) against 2 789 ms for
 * the torch loop of export_state / top-W / import_state / jss_step on the same N*W envs and 205 ms for one
 * jss_step_greedy per round; ta01 at G = 4 096, W = 8 34.9 against 286 ms (DESIGN.md section 4). */
int jss_beam_step(jss_t *h, const float *logits_dev, int64_t ld, int width, float *score_dev, int32_t *parent_out_dev,
                  int32_t *action_out_dev, int32_t *bad_out_dev, void *stream);

/* One round of stochastic beam search (Kool, van Hoof, Welling, ICML 2019) for a policy that reads the observation at
 * every decision: the per-round form of jss_sample_without_replacement(), as jss_beam_step() is of jss_beam_search().
 * Run over a whole search, each group's W slots end as W distinct episodes drawn without replacement from the policy.
 *   Everything is as in jss_beam_step(): groups, live slots, rows, bad rows, the forced no-ops, untouched groups,
 *     parent_out_dev / action_out_dev / bad_out_dev and what a written slot's state and rows equal.  On top of that:
 *   Keys: key_dev, caller-owned fp32 [N], is read and written like score_dev (a search starts with key = [0, -inf, ...,
 *     -inf] per group).  score_dev carries each slot's log-probability under the rows, key_dev its perturbed one.
 *   Noise: group g hashes h = jss_hash3(seed, env_id_base / width + g, step_index), and candidate j of the beam in
 *     slot b gets G_j = (score_b + logp_j) + g_j, g_j the Gumbel noise of h at index b * 256 + j.  With Z = max G,
 *     the candidate at Z (lowest job on ties) gets key T_b, every other one min(T_b, T_b - max(v, 0) - log1p(e^-|v|)),
 *     v = T_b - G_j + log(1 - e^(G_j - Z)): jss_sample_without_replacement()'s arithmetic in its order.  The W best
 *     candidates by key (descending, then parent slot, then job) become the new slots, each with its score and key; an
 *     empty slot gets -inf in both, a failed step NaN in the score.
 *   Rows gathered from a table at each slot's todo, with step_index c + r in round r, give
 *     jss_sample_without_replacement() of that table at counter c on a G-env batch with env_id_base / width bit for
 *     bit (its log_prob is the score here).  Group ids make sharding free: shards with env_id_base = r * N equal the
 *     unsharded batch.
 *   Returns JSS_ERR_INVALID for everything jss_beam_step() rejects, a NULL or not 4-byte-aligned key_dev, and
 *     env_id_base not a multiple of width; JSS_ERR_STATE before jss_assign().
 * Measured on an H100 SXM 80 GB HBM3 at a 700 W power limit with a linear policy on real_obs in torch (median of three
 * rounds): ta80 at G = 256, W = 16 from reset 269 ms per search (135 us per round, policy included) against 220 ms for
 * jss_beam_step() and 190 ms for one jss_step_logits() per round on the same N*W envs; ta01 at G = 4 096, W = 8 41.1
 * against 35.1 and 29.4 ms (DESIGN.md section 4). */
int jss_stochastic_beam_step(jss_t *h, const float *logits_dev, int64_t ld, int width, uint64_t seed,
                             uint64_t step_index, float *score_dev, float *key_dev, int32_t *parent_out_dev,
                             int32_t *action_out_dev, int32_t *bad_out_dev, void *stream);

/* The teacher-forced log-likelihood of k given operation orders per env under a caller's logit table, each from the
 * env's current state, in one launch per lane class present, leaving the envs untouched.
 *   order_dev: device int32 [N][k][jobs_max][machines_max].  Order s of env i stands for the episode that
 *     jss_rollout_priority() on the table -order[i][s] runs from env i's current state: the legal job with the smallest
 *     entry at its current operation, ties to the lowest index, the no-op only when no job is legal.  The orders of
 *     jss_beam_search() and jss_sample_without_replacement() are such tables.
 *   Table: that of jss_rollout_priority_sample().  log_prob_out_dev[i*ld + s] (fp32) is the sum of the episode's
 *     decisions' log-probabilities under it, each computed as jss_rollout_priority_sample() computes the log-probability
 *     of the job it draws; forced no-ops add 0.  NaN where a decision meets a bad row (the episode stops there).
 *     makespan_out_dev[i*ld + s] (int32) is the end time if the episode ends done, else -1.  An env done at entry reads
 *     -1 / 0.  No RNG, no side effects (those of jss_lookahead()).
 *   Returns JSS_ERR_INVALID for a NULL or not 4-byte-aligned pointer, a negative stride, k < 1 or ld < k; JSS_ERR_STATE
 *     before jss_assign(). */
int jss_order_log_prob(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                       const int32_t *order_dev, int64_t k, int32_t *makespan_out_dev, float *log_prob_out_dev,
                       int64_t ld, void *stream);

/* The gradient of jss_order_log_prob(): adds sum_s weights_dev[i*ld + s] * d log_prob[i][s] / d table into grad_out_dev,
 * device fp32 [split][N][jobs_max][machines_max], with jss_sample_episodes_grad()'s accumulator and chunking: chunk c
 * takes the orders s = c (mod split), deterministic for a given split, no atomics.  Orders of weight 0, orders whose
 * episode meets a bad row and envs done at entry add nothing.  Returns JSS_ERR_INVALID as jss_order_log_prob() does and
 * for a split outside 1..k. */
int jss_order_log_prob_grad(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                            const int32_t *order_dev, int64_t k, const float *weights_dev, int64_t ld, int split,
                            float *grad_out_dev, void *stream);

/* jss_order_log_prob() with each order's policy entropy: entropy_out_dev[i*ld + s] (device fp32) is the fp32 sum over
 * the order's decisions of H_t, computed by the helper of jss_rollout_priority_sample_entropy() on the same values, so
 * that an order and a sampled episode drawing the same jobs from the same state report the same entropy bit for bit;
 * forced no-ops add 0, 0 for an env done at entry, NaN where log_prob is NaN.  makespan_out_dev and log_prob_out_dev
 * are bit for bit jss_order_log_prob()'s.  Returns the errors of jss_order_log_prob(), entropy_out_dev checked as its
 * outputs are. */
int jss_order_log_prob_entropy(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                               const int32_t *order_dev, int64_t k, int32_t *makespan_out_dev, float *log_prob_out_dev,
                               float *entropy_out_dev, int64_t ld, void *stream);

/* The gradient of jss_order_log_prob_entropy(): one replay adding sum_s (weights[i*ld + s] * d log_prob[i][s] / d table
 * + entropy_weights[i*ld + s] * d entropy[i][s] / d table) into grad_out_dev, as jss_sample_episodes_entropy_grad() adds
 * it.  Returns the errors of jss_order_log_prob_grad(), entropy_weights_dev checked as weights_dev is. */
int jss_order_log_prob_entropy_grad(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                                    const int32_t *order_dev, int64_t k, const float *weights_dev,
                                    const float *entropy_weights_dev, int64_t ld, int split, float *grad_out_dev,
                                    void *stream);

/* Local search on given operation orders: each of the k orders per env improved by steepest descent on the critical
 * path (the N1 neighbourhood of van Laarhoven, Aarts and Lenstra, 1992: swaps of two adjacent operations of a critical
 * machine block), each from the env's current state, in one launch per lane class present, leaving the envs untouched.
 * No RNG, no logit table.  For each env i and order s (order_dev: device int32 [N][k][jobs_max][machines_max]):
 *   1. Replay: order O stands for the episode jss_order_log_prob() / jss_rollout_priority(-O) runs from env i's state:
 *      the legal job whose current operation has the smallest entry (compared as fp32 of -entry), ties to the lowest
 *      job, the no-op only when no job is legal; at most 2*J_i*M_i + 1 decisions.  The replay records for each
 *      operation it allocates its round (0, 1, ... counting job allocations only) and its start time.
 *   2. Canonical order: R(O)[j][k] is the round of operation (j, k), -1 for operations started before the call.
 *      Replaying R(O) reproduces the episode exactly.  The descent starts from R(O).
 *   3. Chain, on the current canonical schedule, over the in-call operations only (end = start + duration): start at
 *      the operation that ends at the makespan (the largest round if several; none: the chain is empty).  At operation
 *      o with start s, let p_m be the operation on o's machine with the largest round below o's and p_j o's job
 *      predecessor if it is in call.  If p_m ends at s, record the pair (p_m, o) and step to p_m; else if p_j ends at s,
 *      step to p_j; else stop.  Neighbour c is the c-th recorded pair, counted from the makespan end.
 *   4. Neighbour of pair (u, v): R with the entries of u and v swapped, valued by the makespan of its replay.
 *   5. Move: the neighbour of smallest makespan (lowest c on ties), accepted only if strictly below the current
 *      makespan; the current order becomes its canonical order.  Stops at a local optimum or after max_moves moves.
 *   Outputs (device int32, row stride ld >= k, 64-bit index arithmetic): makespan_out_dev[i*ld + s] the final makespan,
 *     start_makespan_out_dev[i*ld + s] the input's, moves_out_dev[i*ld + s] the accepted moves, and
 *     order_out_dev[i][s][j][k] the final canonical order in jss_beam_search()'s format (entries past J_i / M_i are not
 *     written).  An env done at entry, and an input whose replay does not end done (an imported state that errs, or
 *     nothing legal), read -1 / -1 / 0 and -1 in every order entry; a neighbour whose replay does not end done is never
 *     accepted.  order_out_dev may equal order_dev (in place); no other two buffers may overlap.
 *   No side effects: those of jss_lookahead().  The call reads only the state blocks and neither needs nor triggers
 *     jss_refresh_obs().  The results do not depend on the grid, the batch order or sharding.
 *   Returns JSS_ERR_INVALID for a NULL or not 4-byte-aligned pointer, k < 1, ld < k, max_moves < 0 or an overlap other
 *     than in place; JSS_ERR_UNSUPPORTED for k >= 2^31; JSS_ERR_STATE before jss_assign().
 * Memory: one CTA per (env, order), with the canonical order, its start times and the chain's pairs in shared memory
 * (24 KB for ta80, 96 KB for 256 x 32).  Bytes per neighbour decision: none beyond the state block loaded once per
 * neighbour (L2) and the shared-memory tables.  Measured on an H100 SXM 80 GB HBM3 at a 700 W power limit (per-env
 * random tables, at most 3 moves, median of three rounds): ta80 at N = 256 from the best beam_search(W = 16) order
 * 167.9 ms per call against 1 330 ms for the host loop of canonical replay, start-time replay, chain walk and
 * jss_order_log_prob() on the padded neighbours per move; ta80 at N = 256, k = 16 1 919 against 19 962 ms; ta01 at
 * N = 4 096 16.3 against 1 276 ms (DESIGN.md section 4). */
int jss_improve_orders(jss_t *h, const int32_t *order_dev, int64_t k, int max_moves, int32_t *order_out_dev,
                       int32_t *makespan_out_dev, int32_t *start_makespan_out_dev, int32_t *moves_out_dev, int64_t ld,
                       void *stream);

/* Host-buffer form of step(): copies actions H2D, steps, copies the results D2H with
 * contiguous DMA, synchronises.  Any output pointer may be NULL.  Host layouts equal the
 * device layouts: mask_host [N][mask_stride] bytes (row i: bytes 0..J_i), obs_host
 * [N][J][7] fp32, scalars_host [N][4] int32 = the 16-byte records
 * {reward (fp32 bits), reward_raw, current_time_step, flags << 8 | done}. */
int jss_step_host(jss_t *h, const int32_t *actions_host, uint8_t *mask_host, float *obs_host,
                  int32_t *scalars_host, void *stream);

/* Pipelined host-buffer stepping (the e2e path).  jss_host_step_begin enqueues, on internal
 * streams, H2D of the actions, the step kernel, D2H of mask + scalar records (small, first) and
 * the D2H of real_obs via a device staging copy, and returns immediately.
 * jss_host_wait(JSS_WAIT_MASK) blocks until mask/scalars of the latest begin have landed (enough
 * for a host policy to choose the next actions); JSS_WAIT_OBS until its observation has landed.
 * A new begin may follow WAIT_MASK while the previous observation is still streaming into ITS host
 * buffer (callers alternate two pinned observation buffers and call WAIT_OBS before reading one).
 * The pipeline is ordered after the work already enqueued on `after_stream` (the caller's stream),
 * and every stream-ordered entry point (those taking a `stream`) orders its stream after the latest
 * begin, observation transfer included, without blocking the host: a device step, export or
 * statistics call made right after a begin acts on the state that begin left. */
#define JSS_WAIT_MASK 1
#define JSS_WAIT_OBS 2       /* observation of the latest begin */
#define JSS_WAIT_OBS_PREV 3  /* observation of the begin before the latest one */
#define JSS_WAIT_WIRE 4      /* packed rows of the latest begin (they precede its fp32 rows on the copy stream) */
int jss_host_step_begin(jss_t *h, const int32_t *actions_host, uint8_t *mask_host, float *obs_host,
                        int32_t *scalars_host, void *after_stream);
int jss_host_wait(jss_t *h, int what);

/* Packed form of the pipelined host-buffer step: instead of the 28 bytes per job of fp32 real_obs, 10 bytes per job
 * cross PCIe -- the INTEGER numerators of the observation columns (jss_env.py:102-111: legal bit,
 * time_until_finish_current_op, todo_time_step, the stale column-4 numerator, idle_time_jobs_last_op,
 * total_idle_time_jobs; column 3 is derivable) -- and jss_host_expand_obs() rebuilds the exact float observation
 * on the host (multi-threaded; same correctly rounded quotients as the device real_obs, bit for bit).
 * wire_host: [N][jss_host_wire_stride()] bytes (pinned).  scalars_host is required (the expansion reads
 * current_time_step from it).  Waiting works as for jss_host_step_begin: JSS_WAIT_OBS* = the wire rows have landed. */
int jss_host_step_begin_packed(jss_t *h, const int32_t *actions_host, uint8_t *mask_host, uint8_t *wire_host,
                               int32_t *scalars_host, void *after_stream);
/* Hybrid: the first n_dma envs ship their observation as final fp32 rows by DMA (obs_host rows [0, n_dma)), the rest as
 * packed rows (wire_host rows [n_dma, N)) to be expanded with jss_host_expand_obs_range(.., n_dma, N) -- PCIe and the
 * host cores work in parallel, each on its share.  obs_host: pinned [N][J][7] fp32 (also the expansion target). */
int jss_host_step_begin_hybrid(jss_t *h, const int32_t *actions_host, uint8_t *mask_host, uint8_t *wire_host,
                               float *obs_host, int n_dma, int32_t *scalars_host, void *after_stream);
int jss_host_expand_obs_range(jss_t *h, const uint8_t *wire_host, const int32_t *scalars_host, float *obs_host,
                              int env_begin, int env_end);
int64_t jss_host_wire_stride(jss_t *h);
/* wire rows + scalar records of one step -> obs_host [N][J][7] fp32 (rows of env i: J_i * 7 floats written). */
int jss_host_expand_obs(jss_t *h, const uint8_t *wire_host, const int32_t *scalars_host, float *obs_host);

/* Host worker pool shared by jss_host_masked_random / jss_host_expand_obs: `threads` workers (0 = the CPUs this
 * process may use, divided by LOCAL_WORLD_SIZE under torchrun); bind_numa_of_device >= 0 binds them (and the calling
 * thread) to the CPUs of that GPU's NUMA node.  Returns the number of CPUs bound (0 = unbound).  Call before first use. */
int jss_host_configure(int threads, int bind_numa_of_device);
int jss_host_threads(void);
/* Cap the SIMD level of jss_host_expand_obs: 0 scalar, 1 AVX2, 2 AVX-512 (default: best available).  For tests. */
int jss_host_set_simd(int level);

/* --- auxiliary ----------------------------------------------------------- */

/* Per-shard statistics (host int64[JSS_STATS_LEN]); synchronises `stream`. */
int jss_stats(jss_t *h, int64_t *out_host, void *stream);

/* Decode the packed device state into the canonical x_* arrays / load it back
 * (snapshot & restore).  env_mask_dev as in jss_reset.
 * The device state holds each job's x_todo in [0, M_i], x_tufco and x_col4 in
 * [0, JSS_MAX_DURATION] and x_idle_last, x_total_idle in [0, 2^24) -- every state
 * reachable from reset fits, since time never exceeds J*M*JSS_MAX_DURATION < 2^24.
 * jss_import_state clamps a value outside its range into it and sets the env's
 * sticky JSS_FLAG_ERROR bit (visible in flags_done right after the import); the
 * call itself still returns JSS_OK. */
int jss_export_state(jss_t *h, void *stream);
int jss_import_state(jss_t *h, const uint8_t *env_mask_dev, void *stream);

/* Host utility with the device policy's RNG: masked-uniform action per env from
 * a host mask of n rows of `width` (= J+1) bytes, `row_stride` bytes apart, for
 * host-side agents and tests (multi-threaded for large batches). */
int jss_host_masked_random(const uint8_t *mask_host, int n, int width, int64_t row_stride, uint64_t seed,
                           uint64_t env_id_base, uint64_t step_index, int32_t *actions_host);

/* Number of kernels this handle has launched so far (bench.py's gpu_launches). */
int64_t jss_launch_count(const jss_t *h);

#ifdef __cplusplus
}
#endif
#endif /* JSS_B200_H */
