// Host/device shared plain-data types of the batched job-shop kernels.
#pragma once
#include <stdint.h>

// ---- packed instance tables (read-only, built by jss_load_instances) ----------
// ops_pool  u16 [J*M]      op = (machine << 11) | duration   (M <= 32, duration <= 2047)
// len_pool  i32 [J]        jobs_length[j] = sum of durations (jss_env.py:87)
// rem_pool  u16 [J*(M+1)]  rem[j][k] = sum of durations of ops k..M-1 (rules MWR/LWR/CR)
#define JSS_OP_SHIFT 11
#define JSS_OP_DMASK 2047u
#define JSS_OP_NONE 0xFFFFFFFFu  // register-only marker "job has no current op" (finished / padding): machine field >= 32

#ifndef JSS_HD   // as in jss_rng.h
#if defined(__CUDACC__)
#define JSS_HD __host__ __device__
#else
#define JSS_HD
#endif
#endif

// ---- lane classes: lane l of an env's warp owns the KJ = 1 << jss_lane_class(J) jobs KJ*l .. KJ*l+KJ-1 ----------
#define JSS_LANE_CLASSES 4   // KJ = 1, 2, 4, 8 for J <= 32, 64, 128, 256; each class has its own kernels
JSS_HD static inline constexpr int jss_lane_class(int J) { return J <= 32 ? 0 : J <= 64 ? 1 : J <= 128 ? 2 : 3; }
// Job slots a lane reserves, max(4, KJ): the state block pads J to a multiple of them and a mask row J + 1, and a
// lane's legal / no-op-blocked bits are two fields of this width (one byte or one 16-bit word per lane).
JSS_HD static inline constexpr int jss_lane_slots(int KJ) { return KJ > 4 ? KJ : 4; }
// Resident CTAs per SM the step kernel of each lane class is built for: 80 registers -> 3 CTAs = 24 warps per SM, and
// 3 x ~45 KB of shared memory (ta80) fit the 228 KB of an SM; at the 64 registers of 4 CTAs the 4-jobs-per-lane kernel
// spills (DESIGN.md section 4).  <= 32 jobs are latency-bound: 4 CTAs at 64 registers.  8 jobs per lane: one CTA.
// The entries do not grow with the class: a kernel that walks classes 0 .. c (the mixed step kernel) fits class c's.
constexpr int JSS_MIN_CTAS[JSS_LANE_CLASSES] = {4, 3, 3, 1};
static_assert(JSS_MIN_CTAS[0] >= JSS_MIN_CTAS[1] && JSS_MIN_CTAS[1] >= JSS_MIN_CTAS[2] &&
              JSS_MIN_CTAS[2] >= JSS_MIN_CTAS[3], "the mixed-batch step kernel takes its last class's entry");

// ---- packed record of one job: the state block and the host wire rows both use it ------------------
// The five per-job integers carry 76 bits, packed into three words (10 bytes):
//   w0  u32  todo | tufco << 6 | col4 << 17          (bits 28..31: the legal bit in a wire record, 0 in the state block)
//   w1  u32  idle_last | (total_idle & 0xff) << 24
//   w2  u16  total_idle >> 8
// todo = todo_time_step_job in [0, M], M <= 32 (padding slots hold M): 6 bits; tufco =
// time_until_finish_current_op_jobs and col4 = the numerator of real_obs[:,4] (stale by design,
// jss_env.py:569-586) are at most one duration, <= 2047: 11 bits each; idle_last = idle_time_jobs_last_op and
// total_idle = total_idle_time_jobs are at most current_time_step, and time only advances to a pending
// machine completion, so t <= sum_op <= 256 * 32 * 2047 < 2^24: 24 bits each.  jss_import_state checks these
// ranges.  Read as little-endian bytes, w1 and w2 are idle_last (bytes 4..6) and total_idle (bytes 7..9).
#define JSS_PACK_TODO_BITS 6
#define JSS_PACK_DUR_BITS 11
#define JSS_PACK_IDLE_BITS 24
#define JSS_PACK_TUFCO_SHIFT JSS_PACK_TODO_BITS
#define JSS_PACK_COL4_SHIFT (JSS_PACK_TUFCO_SHIFT + JSS_PACK_DUR_BITS)
#define JSS_PACK_LEGAL_SHIFT (JSS_PACK_COL4_SHIFT + JSS_PACK_DUR_BITS)   // wire records only
#define JSS_PACK_W0_MASK ((1u << JSS_PACK_LEGAL_SHIFT) - 1u)   // w0 without a wire record's legal bit
#define JSS_PACK_TODO_MASK ((1u << JSS_PACK_TODO_BITS) - 1u)
#define JSS_PACK_DUR_MASK ((1u << JSS_PACK_DUR_BITS) - 1u)
#define JSS_PACK_IDLE_MAX ((1 << JSS_PACK_IDLE_BITS) - 1)   // largest idle_last / total_idle a record holds

struct JssJobWords {
    uint32_t w0, w1, w2;
};
JSS_HD static inline JssJobWords jss_pack_job(int todo, int tufco, int col4, int idle_last, int total_idle) {
    const uint32_t ti = (uint32_t)total_idle;
    JssJobWords r;
    r.w0 = (uint32_t)todo | ((uint32_t)tufco << JSS_PACK_TUFCO_SHIFT) | ((uint32_t)col4 << JSS_PACK_COL4_SHIFT);
    r.w1 = (uint32_t)idle_last | (ti << JSS_PACK_IDLE_BITS);
    r.w2 = ti >> (32 - JSS_PACK_IDLE_BITS);
    return r;
}
JSS_HD static inline int jss_job_todo(uint32_t w0) { return (int)(w0 & JSS_PACK_TODO_MASK); }
JSS_HD static inline int jss_job_tufco(uint32_t w0) { return (int)((w0 >> JSS_PACK_TUFCO_SHIFT) & JSS_PACK_DUR_MASK); }
// col4 is the top field of a state-block w0; a wire record's w0 goes through JSS_PACK_W0_MASK first
JSS_HD static inline int jss_job_col4(uint32_t w0) { return (int)(w0 >> JSS_PACK_COL4_SHIFT); }
JSS_HD static inline uint32_t jss_job_legal(uint32_t w0) { return w0 >> JSS_PACK_LEGAL_SHIFT; }
JSS_HD static inline int jss_job_idle_last(uint32_t w1) { return (int)(w1 & (uint32_t)JSS_PACK_IDLE_MAX); }
JSS_HD static inline int jss_job_total_idle(uint32_t w1, uint32_t w2) {
    return (int)((w1 >> JSS_PACK_IDLE_BITS) | (w2 << (32 - JSS_PACK_IDLE_BITS)));
}

// ---- per-env state block in HBM (every region 16-byte aligned) -------------------
//   w0  u32[Jcap], w1  u32[Jcap], w2  u16[Jcap] (region padded to a multiple of 16 bytes): the job records
//   tail:  [0, Mcap)  time_until_available_machine (int32)
//   then 2 * slots words (slots = jss_lane_slots(KJ)), byte / 16-bit word l = lane l's job bits: bit i legal(job
//                   KJ*l+i), bit slots+i blocked by a no-op (action_illegal_no_op)
//        4 words  header: current_time_step, flags, episode_steps, episode_return_raw
// Jcap / Mcap are those of the ENV'S OWN instance (jss_block_geom), not batch maxima.
// Not stored because derivable (SURVEY.md section 8 a13): event queue, illegal_actions
// [M][J], machine_legal, both counters, needed_machine_jobs, total_perform_op_time_jobs.
#define JSS_HDR_T 0
#define JSS_HDR_FLAGS 1
#define JSS_HDR_EP_STEPS 2
#define JSS_HDR_EP_RETURN 3

// State-block geometry of an instance in int32 words: the ONE definition the host (block offsets, shared-memory
// sizing, JssInst) and the kernels use.  Per-lane slices are whole vectors: J rounded up to the lane's job slots.
struct JssBlockGeom {
    int32_t Jcap, Mcap;
    int32_t tail;    // first word of tuam (behind w0, w1 and the padded u16 region w2)
    int32_t hdr;     // first word of the 4-word header
    int32_t words;   // whole block
};
JSS_HD static inline JssBlockGeom jss_block_geom(int J, int M) {
    const int slots = jss_lane_slots(1 << jss_lane_class(J));
    JssBlockGeom g;
    g.Jcap = (J + slots - 1) & ~(slots - 1);
    g.Mcap = (M + 3) & ~3;
    g.tail = 2 * g.Jcap + ((g.Jcap + 7) & ~7) / 2;
    g.hdr = g.tail + g.Mcap + 2 * slots;
    g.words = g.hdr + 4;
    return g;
}

// One instance, filled once by jss_load_instances: the kernels stage it in shared memory next to the tables
// (CTA-uniform, re-read with cheap broadcast LDS instead of pinning ~14 registers per thread), or -- uniform batches
// -- read it from the kernel parameters so its fields become constant-bank operands.  The host's packed-row expansion
// divides by the same divisors and reciprocals, so its observation equals the device's bit for bit.
struct JssInst {
    int J, M, max_time_op, max_time_jobs, sum_op;   // jss_env.py:86-89
    float f_mto, f_mtj, f_sop, f_M;       // the divisors as floats ...
    float r_mto, r_mtj, r_sop, r_M;       // ... and their correctly rounded reciprocals (jss_div)
    int Jcap, Mcap, block_words;          // state-block geometry of THIS instance (jss_block_geom) ...
    int tail;                             // ... and the word where tuam starts
    int ops_off, len_off, rem_off;        // offsets into the pools, in elements
};
static_assert(sizeof(JssInst) % 16 == 0, "JssInst is staged with 16-byte copies and keeps the tables behind it aligned");

struct JssTile {       // one CTA work item: up to `count` envs of ONE instance (one 16-byte load)
    int32_t first;     // index into `order`
    int32_t inst_count;  // (instance << 8) | count
    // The state blocks are stored in TILE order with the block size of the env's own instance (a mixed batch
    // moves 272 B for a 15x15 env and 1 136 B for a 100x20 env, not the batch maximum): warp w of this tile
    // owns the block at 16-byte unit  state_off16 + w * block16.
    uint32_t state_off16;
    uint32_t block16;  // block size of this tile's instance in 16-byte units
};

struct JssCtaRange {   // mixed batches: the tiles of one persistent CTA -- an equal slice of EVERY lane class
    int32_t tiles[JSS_LANE_CLASSES][2];   // [tiles[c][0], tiles[c][1]): its tiles of class c (one 8-byte load each)
};

struct JssParams {
    int32_t n_envs;
    // Unused: keeps the kernel-parameter offsets.  Without it ptxas allocates the 80-register mixed-batch step
    // kernels differently and the masked-random one spills; a build with that spill ran cfg5's masked-random step
    // 1.6 % slower on an H100 SXM (400 W power limit).
    int32_t pad0_[3];
    int32_t jobs_max, machines_max, mask_stride, create_flags;
    int32_t uniform_inst;    // >= 0: every env runs this instance and `order` is the identity
    uint64_t env_id_base;
    const JssInst *inst;
    const uint16_t *ops_pool;
    const int32_t *len_pool;
    const uint16_t *rem_pool;
    const int32_t *order;    // env ids grouped by (KJ class, instance)
    const JssTile *tiles;
    const JssCtaRange *cta_ranges;   // mixed-batch step kernel: per CTA an equal slice of every lane class
    int32_t n_cta_ranges;
    int32_t *state;          // per-env blocks of jss_block_geom(J_i, M_i).words words (the env's own instance)
    uint8_t *mask;           // [N][mask_stride]
    float *obs;              // [N][jobs_max][7]
    int32_t *scalars;        // [N][4]: reward (f32 bits), raw reward, current_time_step, flags << 8 | done
    int32_t *solution;       // [N][jobs_max][machines_max] or nullptr
    int32_t *episode_count;
    int32_t *last_makespan;
    int32_t *last_return;
    int64_t *acc;            // [N][4]: total finished-episode steps, sum makespan, sum return, (min<<32|max) packed
    // canonical export buffers
    int32_t *x_todo, *x_tufco, *x_idle_last, *x_total_idle, *x_col4, *x_tuam;
    uint8_t *x_legal, *x_blocked;
};

// A caller's (N, J, M) float table: env i's entry for operation k of job j is at p + i ld_env + j ld_job + k ld_op
// (jss_table_row, jss_table_at).  Priorities or logits, whichever the mode reads.
struct JssTable {
    const float *p;
    int64_t ld_env, ld_job, ld_op;
};

// Per-launch arguments.  Each field holds one thing in every mode that reads it; an entry point sets its mode's fields
// and leaves the rest zero.  Row i of a per-env output starts at i * out_ld.  The fields up to rows_ld include all
// that the fused step kernels read, at byte offsets that jss_device.cuh pins.
struct JssLaunch {
    int32_t tile_begin, tile_end;   // the tiles (jss_beam_step: the group records) of one launch, set by launch_all
    int32_t mode;            // JSS_MODE_*
    int32_t rule;            // JSS_RULE_*: jss_step_sample, jss_policy, jss_rollout (_traj), jss_lookahead
    int32_t coin_mode;       // JSS_COIN_*: the same entry points
    int32_t n_steps;         // the decision budget per env: jss_rollout (_traj), jss_rollout_priority (_sample)
    int32_t write_obs;       // jss_rollout (_traj): emit the observation of every step that changes the env
    int32_t export_after;    // jss_step_export: also decode the new state into the x_* arrays (facade)
    uint64_t explore_t;      // jss_step_greedy (_record): explore iff jss_hash_env(h_env, 0) < explore_t (<= 2^32)
    uint64_t step_index;     // jss_hash3's counter: jss_policy, jss_rollout (_traj), jss_lookahead
    uint32_t hash_key;       // jss_hash_key(seed, step_index): jss_step_sample, jss_step_logits / _greedy (_record)
    int32_t stage;           // JSS_STAGE_*: the instance tables the launch stages in shared memory (launch_all)
    double cr_factor;        // CriticalRatio due_date_factor (dispatching.py:337-349): the entry points that take a rule
    const int32_t *actions;  // [N] the actions a step takes: jss_step (_export), jss_step_sample
    int32_t *actions_out;    // [N] the chosen or next actions: jss_policy, jss_step_sample, jss_step_logits / _greedy
    const uint8_t *env_mask; // [N] the envs a reset or import touches (NULL: all): jss_reset, jss_import_state
    float *traj_obs;         // the caller's slot: jss_rollout_traj (step k of env e at k * n_envs + e), the _record steps
    uint8_t *traj_mask;      // (env e at row e)
    int32_t *traj_scalars;
    int32_t *traj_actions;   // jss_rollout_traj (may be NULL)
    uint8_t *wire;           // [N][wire_stride] packed observation rows (JSS_WIRE_JOB_BYTES per job): pack
    int32_t wire_stride;
    JssInst uni;             // the single instance of a uniform batch (step kernel scalars, tile block size): launch_all
    const float *rows;       // env i's row at rows + i * rows_ld: jss_step_logits / _greedy (_record), jss_beam_step
    float *log_prob_out;     // log-probabilities: the row steps (may be NULL) and the sampling and order modes
    int64_t rows_ld;
    int32_t greedy;          // a row step decodes epsilon-greedily instead of drawing: jss_step_greedy (_record)
    int32_t split;           // S, the work items a tile's candidates or samples are spread over: mode_grid or the caller
    int32_t n_samples;       // K, the samples or orders per env: jss_sample_episodes, jss_order_log_prob (_grad), ...
    int32_t beam_width;      // W, the beams per env (beam search, SWOR) or the envs per group (the beam steps)
    int32_t max_moves;       // the moves each order may take: jss_improve_orders
    uint32_t seed_folded;    // jss_fold32(seed), hashed with sample_counter + d: the table samplers, the stochastic
                             // beam step
    uint64_t seed;           // jss_hash3's seed: jss_policy, jss_rollout (_traj), jss_lookahead
    uint64_t sample_counter; // the RNG counter of an env's first draw (jss_stochastic_beam_step: of the round)
    int64_t out_ld;          // the row stride of every per-env output row, and of the weights
    JssTable table;          // the caller's table: the priority, sampling, beam-search and order modes
    const int32_t *order_in;     // [N][K][jobs_max][machines_max] orders: jss_order_log_prob (_grad), jss_improve_orders
    const int32_t *sample_in;    // [N] the sample each env replays (< 0: none): jss_sample_episodes_solution
    const float *weights;        // row i: each sample's weight: the _grad modes
    uint16_t *beam_trace;        // per CTA, W backpointers per round: the beam searches that write orders (NULL: none)
    const int32_t *beam_groups;  // per group [g, instance, W block offsets in 16-byte units], by lane class: beam steps
    int32_t *values_out;     // row i: each action's value: jss_lookahead (_priority; _sample: K per action)
    int32_t *makespan_out;   // row i: each sample's, slot's or order's makespan
    float *score_out;        // row i: each slot's score: jss_beam_search
    float *key_out;          // row i: each slot's key: jss_sample_without_replacement
    int32_t *start_out;      // row i: each input order's makespan: jss_improve_orders
    int32_t *moves_out;      // row i: each order's accepted moves: jss_improve_orders
    int32_t *order_out;      // [jobs_max][machines_max] per order written: the beam searches (may be NULL), improve
    int32_t *solution_out;   // [N][jobs_max][machines_max] start times: jss_sample_episodes_solution
    float *grad_out;         // [N][jobs_max][machines_max] per chunk: jss_rollout_priority_sample (may be NULL), _grad
    float *score_io;         // [N] each slot's score, read and written: the beam steps (slot b of group g: env g W + b)
    float *key_io;           // [N] each slot's key, read and written: jss_stochastic_beam_step
    int32_t *parent_out;     // [N] each slot's parent slot: the beam steps
    int32_t *job_out;        // [N] each slot's job: the beam steps
    int32_t *bad_out;        // [N / W] each group's bad-row bit: the beam steps
    float *entropy_out;      // the entropy of each episode, beside log_prob_out: the _ENT modes
    float *entropy_grad_out; // [N][jobs_max][machines_max] d entropy / d table: jss_rollout_priority_sample_entropy
                             // (may be NULL)
    const float *entropy_weights;   // row i: each sample's weight of the entropy gradient: the _ENT_GRAD modes
};

#define JSS_MODE_RESET 0
#define JSS_MODE_STEP 1
#define JSS_MODE_ROLLOUT 2
#define JSS_MODE_POLICY 3
#define JSS_MODE_EXPORT 4
#define JSS_MODE_IMPORT 5
#define JSS_MODE_PACK 6     // packed observation wire rows for the host-buffer path (jss_host_step_begin_packed)
#define JSS_MODE_REFRESH 7  // rewrite real_obs from the state blocks (jss_refresh_obs)
#define JSS_MODE_PRIORITY 8 // run each env to the end of its episode on a caller's priority table (jss_rollout_priority)
#define JSS_MODE_PRIORITY_SAMPLE 9   // the same, each decision drawn from a softmax over the table's entries
                                     // (jss_rollout_priority_sample)
#define JSS_MODE_LOOKAHEAD 10        // each legal action's makespan under a rule's rollout, the envs untouched
                                     // (jss_lookahead)
#define JSS_MODE_LOOKAHEAD_PRIORITY 11   // the same under the greedy decisions of a caller's priority table
                                         // (jss_lookahead_priority)
#define JSS_MODE_SAMPLE_EPISODES 12      // K episodes per env drawn from a logit table, the envs untouched
                                         // (jss_sample_episodes)
#define JSS_MODE_SAMPLE_EPISODES_GRAD 13       // their replay, adding the weighted gradients into the caller's
                                               // chunks (jss_sample_episodes_grad)
#define JSS_MODE_SAMPLE_EPISODES_SOLUTION 14   // the replay of one sample per env, writing the start times
                                               // (jss_sample_episodes_solution)
#define JSS_MODE_BEAM_SEARCH 15          // beam search over a logit table, one env per CTA, the envs untouched
                                         // (jss_beam_search)
#define JSS_MODE_SWOR 16                 // the same perturbed by top-down Gumbel noise: W distinct episodes drawn
                                         // without replacement (jss_sample_without_replacement)
#define JSS_MODE_ORDER_LOG_PROB 17       // the log-likelihood of K given operation orders per env under a logit
                                         // table, the envs untouched (jss_order_log_prob)
#define JSS_MODE_ORDER_LOG_PROB_GRAD 18  // its weighted gradient, added into the caller's chunks
                                         // (jss_order_log_prob_grad)
#define JSS_MODE_BEAM_STEP 19            // one beam-search round per group of W envs from per-beam logit rows, the
                                         // children stepped into the group's envs (jss_beam_step)
#define JSS_MODE_STOCHASTIC_BEAM_STEP 20 // the same perturbed by top-down Gumbel noise, the beams ranked by key
                                         // (jss_stochastic_beam_step)
#define JSS_MODE_IMPROVE_ORDERS 21       // operation orders improved by steepest descent on the critical path, one
                                         // (env, order) per CTA, the envs untouched (jss_improve_orders)
#define JSS_MODE_LOOKAHEAD_SAMPLE 22     // each legal action's makespans under K episodes drawn from a logit table
                                         // after it, the envs untouched (jss_lookahead_sample)
// The entropy forms of the three differentiable log-probability producers: each also writes every episode's policy
// entropy, the fp32 sum over its decisions of H_t = log S - T / S (jss_softmax_entropy), into a.entropy_out.
#define JSS_MODE_PRIORITY_SAMPLE_ENT 23  // JSS_MODE_PRIORITY_SAMPLE, with d entropy / d table into a.entropy_grad_out
                                         // (jss_rollout_priority_sample_entropy)
#define JSS_MODE_SAMPLE_EPISODES_ENT 24  // JSS_MODE_SAMPLE_EPISODES (jss_sample_episodes_entropy)
#define JSS_MODE_SAMPLE_EPISODES_ENT_GRAD 25   // its replay, adding w_s G_lp + v_s G_H with v_s from
                                               // a.entropy_weights (jss_sample_episodes_entropy_grad)
#define JSS_MODE_ORDER_LOG_PROB_ENT 26   // JSS_MODE_ORDER_LOG_PROB (jss_order_log_prob_entropy)
#define JSS_MODE_ORDER_LOG_PROB_ENT_GRAD 27    // its gradient as JSS_MODE_SAMPLE_EPISODES_ENT_GRAD's
                                               // (jss_order_log_prob_entropy_grad)
#define JSS_NUM_MODES 28                 // the rows of JSS_MODES (jss_device.cuh)

#define JSS_WARPS_PER_CTA 8
