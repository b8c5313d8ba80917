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

struct JssLaunch {           // per-launch arguments
    int32_t tile_begin, tile_end;
    int32_t mode;            // JSS_MODE_*
    union {
        int32_t rule;
        int32_t greedy;      // steps from a row (a.logits): 0 categorical draw, 1 epsilon-greedy decode
        int32_t n_samples;   // jss_sample_episodes (_grad): K, the episodes drawn per env; jss_order_log_prob (_grad),
                             // jss_improve_orders: K, the orders per env
        int32_t beam_width;  // jss_beam_search, jss_sample_without_replacement: W, the beams kept per env;
                             // jss_beam_step, jss_stochastic_beam_step: W, the envs per group
    };
    int32_t coin_mode, n_steps, write_obs;   // jss_lookahead (_priority): n_steps is S, the work items each tile's
                                             // candidates are spread over (launch_all); jss_sample_episodes: the
                                             // work items each tile's samples are spread over (_grad: the chunks)
    int32_t export_after;    // step through the generic kernel: also decode the new state into the x_* arrays (facade)
    union {
        uint64_t seed;
        uint64_t explore_t;  // epsilon-greedy decode: an env explores iff jss_hash_env(h_env, 0) < explore_t, 0 .. 2^32
        int64_t prio_ld_job; // jss_rollout_priority: element stride between jobs of the priority table
    };
    union {
        uint64_t step_index;
        int64_t prio_ld_op;  // jss_rollout_priority: element stride between operations of a job
    };
    uint32_t hash_key;       // jss_hash_key(seed, step_index), folded once per launch on the host (fused step + sampler);
                             // jss_rollout_priority_sample: jss_fold32(seed), all of the seed that jss_hash3 reads
    int32_t stage;           // JSS_STAGE_*: the instance tables the launch stages in shared memory (launch_all)
    union {
        double cr_factor;    // CriticalRatio due_date_factor (dispatching.py:337-349); reference default 1.5
        uint64_t sample_step_index;   // jss_rollout_priority_sample: the RNG counter of the env's first decision
                                      // (jss_stochastic_beam_step: of the round)
        int64_t values_ld;   // jss_lookahead_priority: env i's value of action a at actions_out + i * values_ld + a
                             // (logits_ld is the table's env stride there)
        const int32_t *order_in;   // jss_order_log_prob (_grad), jss_improve_orders: order s of env i at order_in +
                                   // (i * n_samples + s) * jobs_max * machines_max
    };
    union {
        const int32_t *actions;  // step; jss_sample_episodes_solution: the sample each env replays (< 0: none)
        const float *weights;    // jss_sample_episodes_grad: sample s of env i weighs weights[i * samples_ld + s]
        uint16_t *beam_trace;    // jss_beam_search with an order: per CTA, W backpointers per round (NULL: no order)
        const int32_t *beam_groups;   // jss_beam_step: per group [group, instance, W block offsets in 16-byte units],
                                      // grouped by lane class; a launch takes records [tile_begin, tile_end)
    };
    union {
        int32_t *actions_out;    // policy; jss_lookahead: env i's value of action a at actions_out + i * logits_ld + a
                                 // (jss_lookahead_priority: + i * values_ld + a); jss_sample_episodes: sample s's
                                 // makespan at actions_out + i * samples_ld + s
        int32_t *solution_out;   // jss_sample_episodes_solution: [N][jobs_max][machines_max] start times
                                 // (jss_beam_search: slot b's makespan at actions_out + i * samples_ld + b)
        int32_t *parent_out;     // jss_beam_step: [N] each slot's parent slot
    };
    union {
        const uint8_t *env_mask; // reset / import
        int64_t samples_ld;      // jss_sample_episodes (_grad): row stride of the per-sample outputs / weights;
                                 // jss_beam_search: of the per-slot outputs
    };
    // rollout with trajectory recording: outputs of step k of env e go to slot k * n_envs + e of these buffers;
    // jss_step_logits_record / jss_step_greedy_record: env e's observation, mask and scalar record go to row e of
    // traj_obs / mask / scalars.  jss_rollout_priority_sample: grad_out is the [N][jobs_max][machines_max] gradient of
    // each env's log-probability with respect to its table entries (may be NULL)
    // jss_beam_search: order_out is the [N][jobs_max][machines_max] order of each env's best slot (may be NULL), and
    // slot b's score goes to log_prob_out + i * samples_ld + b
    // jss_beam_step: slot b of group g has score log_prob_out[g W + b] (read and written), parent parent_out, job
    // job_out, and group g's bad-row bit goes to bad_out[g]
    union {
        float *traj_obs;
        float *grad_out;
        int32_t *order_out;
        int32_t *job_out;
    };
    // jss_stochastic_beam_step: as jss_beam_step, and slot b of group g has key key_io[g W + b] (read and written)
    // jss_improve_orders: order s of env i goes to order_out + (i * n_samples + s) * jobs_max * machines_max, its
    // makespan to actions_out, the input's to start_out and the accepted moves to moves_out, each at i * samples_ld + s;
    // n_steps is the move limit
    union {
        uint8_t *traj_mask;
        float *key_io;
        int32_t *moves_out;
    };
    int32_t *traj_scalars; int32_t *traj_actions;
    // jss_sample_without_replacement: slot b's score goes to log_prob_out and its key to key_out + i * samples_ld + b,
    // and order_out is the [N][W][jobs_max][machines_max] order of every slot (may be NULL)
    union {
        uint8_t *wire;       // pack: [N][wire_stride] packed observation rows (JSS_WIRE_JOB_BYTES per job)
        float *key_out;
        int32_t *bad_out;
        int32_t *start_out;
    };
    int32_t wire_stride;
    JssInst uni;             // the single instance of a uniform batch (step kernel scalars, tile block size)
    // jss_step_logits / jss_step_greedy: env i's logits (scores) at logits + i * logits_ld; the chosen actions go to
    // actions_out, their log-probabilities to log_prob_out (may be NULL).  jss_rollout_priority (_sample): env i's
    // priority (logit) of operation k of job j at logits + i * logits_ld + j * prio_ld_job + k * prio_ld_op; _sample
    // writes env i's episode log-probability to log_prob_out[i]
    const float *logits;
    float *log_prob_out;
    int64_t logits_ld;
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
#define JSS_NUM_MODES 22                 // the rows of JSS_MODES (jss_device.cuh)

#define JSS_WARPS_PER_CTA 8
