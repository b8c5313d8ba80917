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

struct JssInstDesc {
    int32_t J, M;
    int32_t max_time_op, max_time_jobs, sum_op;  // jss_env.py:86-89
    int32_t ops_off;                              // offsets into the pools, in elements
    int32_t len_off;
    int32_t rem_off;
    // correctly rounded fp32 reciprocals of the four observation divisors (jss_div)
    float r_mto, r_mtj, r_sop, r_M;
};

#ifndef JSS_HD   // as in jss_rng.h
#if defined(__CUDACC__)
#define JSS_HD __host__ __device__
#else
#define JSS_HD
#endif
#endif

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
//   then 8 words  = 32 bytes, byte l = lane l's job bits: bit i legal(job KJ*l+i),
//                   bit 4+i blocked by a no-op (action_illegal_no_op)
//                   (instances with 129..256 jobs, KJ = 8: 16 words, one 16-bit word per lane, blocked = bit 8+i)
//        4 words  header: current_time_step, flags, episode_steps, episode_return_raw
// Jcap / Mcap are those of the ENV'S OWN instance (jss_block_geom), not batch maxima.
// Not stored because derivable (SURVEY.md section 8 a13): event queue, illegal_actions
// [M][J], machine_legal, both counters, needed_machine_jobs, total_perform_op_time_jobs.
#define JSS_HDR_T 0
#define JSS_HDR_FLAGS 1
#define JSS_HDR_EP_STEPS 2
#define JSS_HDR_EP_RETURN 3

// State-block geometry of an instance in int32 words: the ONE definition the host (block offsets, shared-memory
// sizing) and the kernels (SmInst) use.  Per-lane slices are whole vectors: J rounded up to 4 (to 8 for the
// 8-jobs-per-lane class, which also keeps 16 bits per lane in the bits region).
struct JssBlockGeom {
    int32_t Jcap, Mcap;
    int32_t tail;    // first word of tuam (behind w0, w1 and the padded u16 region w2)
    int32_t hdr;     // first word of the 4-word header
    int32_t words;   // whole block
};
JSS_HD static inline JssBlockGeom jss_block_geom(int J, int M) {
    JssBlockGeom g;
    g.Jcap = J > 128 ? ((J + 7) & ~7) : ((J + 3) & ~3);
    g.Mcap = (M + 3) & ~3;
    g.tail = 2 * g.Jcap + ((g.Jcap + 7) & ~7) / 2;
    g.hdr = g.tail + g.Mcap + (J > 128 ? 16 : 8);
    g.words = g.hdr + 4;
    return g;
}

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
    int32_t a4, b4, a2, b2;     // [a4, b4) KJ = 4 tiles, [a2, b2) KJ = 2 tiles,
    int32_t a1, b1, a8, b8;     // [a1, b1) KJ = 1 tiles, [a8, b8) KJ = 8 tiles (instances with 129..256 jobs)
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
    const JssInstDesc *inst;
    const uint16_t *ops_pool;
    const int32_t *len_pool;
    const uint16_t *rem_pool;
    const int32_t *order;    // env ids grouped by (KJ class, instance)
    const JssTile *tiles;
    const JssCtaRange *cta_ranges;   // mixed-batch step kernel: per CTA an equal slice of every lane class
    int32_t n_cta_ranges;
    const uint32_t *state_off16;   // per env: start of its state block, in 16-byte units (tile order, see JssTile)
    const uint32_t *hdr_off16;     // per env: start of its 4-word header (t, flags, episode steps / return), 16-byte units
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

// Per-instance scalars: staged in shared memory next to the tables (CTA-uniform, re-read with cheap
// broadcast LDS instead of pinning ~14 registers per thread), or -- uniform batches -- passed in the
// kernel parameters so they become constant-bank operands.
struct SmInst {
    int J, M, max_time_op, max_time_jobs, sum_op;
    float f_mto, f_mtj, f_sop, f_M;       // the divisors as floats ...
    float r_mto, r_mtj, r_sop, r_M;       // ... and their correctly rounded reciprocals
    int Jcap, Mcap, block_words;          // state-block geometry of THIS instance (jss_block_geom) ...
    int tail;                             // ... and the word where tuam starts
    int pad_[3];                          // 20 words: the tables behind it in shared memory stay 16-byte aligned
};
static_assert(sizeof(SmInst) % 16 == 0, "SmInst must keep the shared-memory tables 16-byte aligned");
struct JssLaunch {           // per-launch arguments
    int32_t tile_begin, tile_end;
    int32_t mode;            // JSS_MODE_*
    int32_t rule, coin_mode, n_steps, write_obs;
    int32_t export_after;    // step through the generic kernel: also decode the new state into the x_* arrays (facade)
    uint64_t seed, step_index;
    uint32_t hash_key;       // jss_hash_key(seed, step_index), folded once per launch on the host (fused step + sampler)
    uint32_t pad_key_;
    double cr_factor;        // CriticalRatio due_date_factor (dispatching.py:337-349); reference default 1.5
    const int32_t *actions;  // step
    int32_t *actions_out;    // policy
    const uint8_t *env_mask; // reset / import
    // rollout with trajectory recording: outputs of step k of env e go to slot k * n_envs + e of these buffers
    float *traj_obs; uint8_t *traj_mask; int32_t *traj_scalars; int32_t *traj_actions;
    uint8_t *wire;           // pack: [N][wire_stride] packed observation rows (JSS_WIRE_JOB_BYTES per job)
    int32_t wire_stride;
    SmInst uni;              // scalars of the single instance of a uniform batch (step kernel, UNI = true)
};

#define JSS_MODE_RESET 0
#define JSS_MODE_STEP 1
#define JSS_MODE_ROLLOUT 2
#define JSS_MODE_POLICY 3
#define JSS_MODE_EXPORT 4
#define JSS_MODE_IMPORT 5
#define JSS_MODE_PACK 6     // packed observation wire rows for the host-buffer path (jss_host_step_begin_packed)

#define JSS_WARPS_PER_CTA 8
