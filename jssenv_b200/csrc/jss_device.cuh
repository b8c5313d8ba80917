// jss_device.cuh -- sm_90a device code of the batched job-shop environment.
//
// One warp simulates one environment.  Lane l owns the KJ = 1, 2, 4 (or, for 129..256 jobs, 8) consecutive jobs
// KJ*l .. KJ*l+KJ-1 (so its slice of every per-job array is ONE 4/8/16-byte vector
// load/store and its slice of real_obs is 7 consecutive vectors), and lane m (< M <= 32)
// owns machine m.  A lane keeps the legal / no-op-blocked bits of its own jobs in one
// register (`lb`: bits 0..3 legal, bits 4..7 blocked); warp-wide facts are obtained with
// single VOTE / REDUX instructions.  Everything the reference keeps redundantly (event
// queue, illegal_actions[M][J], machine_legal, counters, needed_machine, total_perform)
// is re-derived in registers (SURVEY.md section 8 a13, appendix A).
//
// Reference semantics implemented here (file:line relative to the reference):
//   env_reset_regs      JSSEnv/envs/jss_env.py:145-181  reset
//   env_advance         JSSEnv/envs/jss_env.py:495-637  increase_time_step
//   env_prioritize      JSSEnv/envs/jss_env.py:183-254  _prioritization_non_final
//   env_check_no_op     JSSEnv/envs/jss_env.py:256-401  _check_no_op
//   env_step            JSSEnv/envs/jss_env.py:403-481  step (+483-493, 639-653)
//   env_emit_*          JSSEnv/envs/jss_env.py:102-134  observation / mask
//   env_select_action   JSSEnv/dispatching.py:92-408    rules; README.md:58-60 sampler
//
// The same source is compiled for the host by tests/emu (32 fibers per warp,
// collectives emulated) so the logic can be differential-tested against the
// oracle without a GPU; that build is test-only and is never loaded by the
// product library.
#pragma once
#include <stdint.h>
#include <string.h>
#include <type_traits>

#include "../../include/jss_b200.h"
#include "jss_rng.h"
#include "jss_types.h"

#define JSS_FULL 0xffffffffu
#define JSS_INF 0x7fffffff

#ifndef JSS_DEV
#define JSS_DEV __device__ __forceinline__
#endif

struct InstView {  // instance tables staged in shared memory
    const uint16_t *ops;
    const int32_t *len;
    const uint16_t *rem;
    const JssInst *si;
    // Shape of the instance for branch conditions and loop bounds.  Uniform-batch kernels point `si` at the kernel
    // parameters (constant bank: ptxas knows those are warp-uniform) and read it there; kernels that stage the instance
    // in shared memory keep register copies that went through jss_uniform (jss_iv_shape).
    int Ju, Mu;
    bool staged;       // compile-time constant after inlining
};
JSS_DEV int jss_J(const InstView &iv) { return iv.staged ? iv.Ju : iv.si->J; }
JSS_DEV int jss_M(const InstView &iv) { return iv.staged ? iv.Mu : iv.si->M; }

template <int KJ>
struct EnvRegs {
    int todo[KJ], tufco[KJ], idle_last[KJ], total_idle[KJ], col4[KJ];
    uint32_t op[KJ];   // packed current op of each owned job, JSS_OP_NONE if none
    uint32_t lb;       // this lane's jobs: bit i = legal, bit 4+i = blocked by a no-op
    int tuam;          // lane m: time_until_available_machine[m]
    int t;             // current_time_step
    uint32_t flags;
    int ep_steps, ep_return;
    // What the step changed of job slot i, for the uniform step kernels' stores, which write back just the 32-byte
    // sectors of the row and of the state block that hold a marked job: bit JSS_DIRTY_W0 + i / W1 + i / W2 + i its
    // word in the block's region w0 / w1 / w2, bit JSS_DIRTY_LEGAL + i its legal bit (column 0 of its row, not in the
    // job record).  Its row changed iff one of the first two or the last is set (env_dirty_rows).
    uint32_t dirty;
};
#define JSS_DIRTY_W0 0
#define JSS_DIRTY_W1 8
#define JSS_DIRTY_W2 16
#define JSS_DIRTY_LEGAL 24
template <int KJ>
JSS_DEV uint32_t env_dirty_rows(const EnvRegs<KJ> &s) {
    return (s.dirty >> JSS_DIRTY_W0) | (s.dirty >> JSS_DIRTY_W1) | (s.dirty >> JSS_DIRTY_LEGAL);
}

// ---- warp-uniformity hints -----------------------------------------------------------
// ptxas proves a warp converged only while every branch on the way depends on values it KNOWS to be warp-uniform
// (kernel parameters, blockIdx, results of vote / redux / a shuffle from a fixed lane).  One branch on a value it
// cannot classify -- threadIdx.x >> 5, a word every lane loaded from the same shared-memory address -- and every
// *_sync collective after it is compiled as "maybe diverged": UMOV + BRA.DIV + an out-of-line WARPSYNC stub per
// collective, BSSY/BSYNC around each branch, nothing kept in uniform registers.  The few truly uniform inputs of an
// env-step go through a lane-0 shuffle.  ptxas for sm_90a still guards the collectives with BRA.DIV, but the hinted
// code is faster where it matters: measured on an H100 SXM (80 GB HBM3, 400 W power limit), the mixed-batch step
// kernel (cfg5, N = 65 536) takes 126.8 / 131.5 us per launch with FIFO / MWR instead of 134.9 / 139.0 us with the
// shuffle left out (6 %); uniform ta80 batches are unchanged (195 us either way).
// The value MUST be the same in every lane -- the shuffle is a hint, not a broadcast of lane 0's opinion.
JSS_DEV int jss_uniform(int v) { return __shfl_sync(JSS_FULL, v, 0); }
JSS_DEV uint32_t jss_uniform(uint32_t v) { return (uint32_t)jss_uniform((int)v); }
JSS_DEV int jss_warp_index() { return jss_uniform((int)(threadIdx.x >> 5)); }
// Where the flags word gets the hint: everywhere except the uniform 4-jobs-per-lane step kernel (the ta71..80 shape),
// which keeps the conservative code (hinting it too has not been measured on H100 in isolation).
template <int KJ, bool UNI>
JSS_DEV constexpr bool jss_hint_flags() { return !(UNI && KJ == 4); }

// ---- small helpers --------------------------------------------------------------
template <int KJ, typename T>
JSS_DEV T jss_sel(const T (&a)[KJ], int i) {  // a[i] without dynamic register indexing
    T r = a[0];
#pragma unroll
    for (int k = 1; k < KJ; k++) r = (i == k) ? a[k] : r;
    return r;
}
// (mask >> pos) & 1 for pos that may be >= 32 (JSS_OP_NONE): the hardware shift clamps,
// the host emulation needs the explicit test
JSS_DEV uint32_t jss_bit(uint32_t mask, uint32_t pos) {
#ifdef JSS_EMU
    return pos < 32u ? (mask >> pos) & 1u : 0u;
#else
    return __funnelshift_rc(mask, 0u, pos) & 1u;   // SHF.R with the shift clamped to 32
#endif
}
JSS_DEV uint32_t jss_op_m(uint32_t op) { return op >> JSS_OP_SHIFT; }
JSS_DEV int jss_op_d(uint32_t op) { return (int)(op & JSS_OP_DMASK); }
template <int KJ>
JSS_DEV constexpr uint32_t jss_legal_mask() { return (1u << KJ) - 1u; }
// `lb` layout: bit i = job slot i legal, bit BS + i = blocked by a no-op, BS = jss_lane_slots(KJ); a lane's bits are
// one byte of the state block (KJ <= 4) or one 16-bit word (KJ = 8: 129..256 jobs)
template <int KJ>
JSS_DEV constexpr int jss_bs() { return jss_lane_slots(KJ); }
template <int KJ>
JSS_DEV constexpr int jss_bits_words() { return 2 * jss_lane_slots(KJ); }   // int32 words of the per-lane bits region

// correctly rounded x / y for small non-negative integers given ry = RN(1/y): Markstein's
// sequence q = RN(x*ry); r = x - q*y (exact, FMA); q' = RN(q + r*ry).  Checked exhaustively
// against IEEE division for every (x, y) the bundled instances can produce and all y <= 4096
// (tools/check_div.c); replaces the ~25-instruction IEEE fp32 division and its slow path.
JSS_DEV float jss_div(float x, float y, float ry) {
    const float q = __fmul_rn(x, ry);
    const float r = __fmaf_rn(-q, y, x);
    return __fmaf_rn(r, ry, q);
}

// ---- TMA (cp.async.bulk) + mbarrier helpers -----------------------------------------------
// The state block of the NEXT env of a warp is prefetched into the warp's shared-memory
// buffer by one bulk copy (global -> shared, completion on an mbarrier) while the current env
// is simulated; an env's observation rows leave shared memory with one bulk copy
// (shared -> global).  Sizes/addresses are multiples of 16 bytes by construction.
// Shared-memory operands are passed as 32-bit shared-space addresses (jss_saddr_t) computed from
// ONE base register, so no generic<->shared address conversions are needed at the call sites.
#ifndef JSS_EMU
typedef uint32_t jss_saddr_t;
JSS_DEV jss_saddr_t jss_saddr(const void *generic_ptr) { return (uint32_t)__cvta_generic_to_shared(generic_ptr); }
JSS_DEV void jss_mbar_init(jss_saddr_t mbar) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mbar) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
JSS_DEV void jss_bulk_load(jss_saddr_t smem_dst, const void *gmem_src, uint32_t bytes, jss_saddr_t mbar) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_dst), "l"(gmem_src), "r"(bytes), "r"(mbar) : "memory");
}
JSS_DEV void jss_mbar_wait(jss_saddr_t mbar, uint32_t phase) {
    uint32_t ok;
    do {
        // non-blocking poll: test_wait returns at once, where try_wait may park the warp for a scheduler time slice
        // when the block has not landed yet
        asm volatile("{\n .reg .pred p;\n mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                     : "=r"(ok) : "r"(mbar), "r"(phase) : "memory");
    } while (!ok);
}
JSS_DEV void jss_fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
JSS_DEV void jss_bulk_store(void *gmem_dst, jss_saddr_t smem_src, uint32_t bytes) {   // joins the open bulk group
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                 ::"l"(gmem_dst), "r"(smem_src), "r"(bytes) : "memory");
}
JSS_DEV void jss_bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
JSS_DEV void jss_bulk_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
JSS_DEV void jss_bulk_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// 4-byte asynchronous copies global -> shared (LDGSTS), per-thread groups: the policy-logits rows of jss_step_logits are
// only 4-byte aligned (an (N, J+1) fp32 tensor has 404-byte rows for ta80), which rules out the bulk copy
JSS_DEV void jss_cp_async4(jss_saddr_t smem_dst, const void *gmem_src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_dst), "l"(gmem_src) : "memory");
}
JSS_DEV void jss_cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
JSS_DEV void jss_cp_async_wait() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
#else   // host emulation (tests/emu): synchronous copies; the waits are warp rendezvous points
typedef char *jss_saddr_t;
JSS_DEV jss_saddr_t jss_saddr(const void *generic_ptr) { return (char *)generic_ptr; }
JSS_DEV void jss_mbar_init(jss_saddr_t) {}
JSS_DEV void jss_bulk_load(jss_saddr_t smem_dst, const void *gmem_src, uint32_t bytes, jss_saddr_t) { memcpy(smem_dst, gmem_src, bytes); }
JSS_DEV void jss_mbar_wait(jss_saddr_t, uint32_t) { __syncwarp(); }
JSS_DEV void jss_fence_async_smem() {}
JSS_DEV void jss_bulk_store(void *gmem_dst, jss_saddr_t smem_src, uint32_t bytes) { memcpy(gmem_dst, smem_src, bytes); }
JSS_DEV void jss_bulk_commit() {}
JSS_DEV void jss_bulk_store_wait_read() {}
JSS_DEV void jss_bulk_store_wait_all() {}
JSS_DEV void jss_cp_async4(jss_saddr_t smem_dst, const void *gmem_src) { memcpy(smem_dst, gmem_src, 4); }
JSS_DEV void jss_cp_async_commit() {}
JSS_DEV void jss_cp_async_wait() {}
#endif

// vector access to a lane's KJ-word slice
template <int KJ>
JSS_DEV void jss_ld(const int32_t *p, int (&o)[KJ]);
template <>
JSS_DEV void jss_ld<1>(const int32_t *p, int (&o)[1]) { o[0] = *p; }
template <>
JSS_DEV void jss_ld<2>(const int32_t *p, int (&o)[2]) {
    int2 v = *reinterpret_cast<const int2 *>(p);
    o[0] = v.x; o[1] = v.y;
}
template <>
JSS_DEV void jss_ld<4>(const int32_t *p, int (&o)[4]) {
    int4 v = *reinterpret_cast<const int4 *>(p);
    o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
}
template <>
JSS_DEV void jss_ld<8>(const int32_t *p, int (&o)[8]) {
    const int4 a = reinterpret_cast<const int4 *>(p)[0], b = reinterpret_cast<const int4 *>(p)[1];
    o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
}
template <int KJ>
JSS_DEV void jss_st(int32_t *p, const int (&o)[KJ]);
template <>
JSS_DEV void jss_st<1>(int32_t *p, const int (&o)[1]) { *p = o[0]; }
template <>
JSS_DEV void jss_st<2>(int32_t *p, const int (&o)[2]) { *reinterpret_cast<int2 *>(p) = make_int2(o[0], o[1]); }
template <>
JSS_DEV void jss_st<4>(int32_t *p, const int (&o)[4]) {
    *reinterpret_cast<int4 *>(p) = make_int4(o[0], o[1], o[2], o[3]);
}

template <>
JSS_DEV void jss_st<8>(int32_t *p, const int (&o)[8]) {
    reinterpret_cast<int4 *>(p)[0] = make_int4(o[0], o[1], o[2], o[3]);
    reinterpret_cast<int4 *>(p)[1] = make_int4(o[4], o[5], o[6], o[7]);
}

// vector access to a lane's KJ-entry slice of a u16 array (2 / 4 / 8 / 16 bytes)
// (two u16 entries per 32-bit word, the lower index in the low half)
template <int KJ>
JSS_DEV void jss_ld16(const uint16_t *p, uint32_t (&o)[KJ]);
template <>
JSS_DEV void jss_ld16<1>(const uint16_t *p, uint32_t (&o)[1]) { o[0] = p[0]; }
template <>
JSS_DEV void jss_ld16<2>(const uint16_t *p, uint32_t (&o)[2]) {
    const uint32_t v = *reinterpret_cast<const uint32_t *>(p);
    o[0] = v & 0xffffu; o[1] = v >> 16;
}
template <>
JSS_DEV void jss_ld16<4>(const uint16_t *p, uint32_t (&o)[4]) {
    const uint2 v = *reinterpret_cast<const uint2 *>(p);
    o[0] = v.x & 0xffffu; o[1] = v.x >> 16; o[2] = v.y & 0xffffu; o[3] = v.y >> 16;
}
template <>
JSS_DEV void jss_ld16<8>(const uint16_t *p, uint32_t (&o)[8]) {
    const uint4 v = *reinterpret_cast<const uint4 *>(p);
    o[0] = v.x & 0xffffu; o[1] = v.x >> 16; o[2] = v.y & 0xffffu; o[3] = v.y >> 16;
    o[4] = v.z & 0xffffu; o[5] = v.z >> 16; o[6] = v.w & 0xffffu; o[7] = v.w >> 16;
}
// o[] < 2^16
template <int KJ>
JSS_DEV void jss_st16(uint16_t *p, const uint32_t (&o)[KJ]);
template <>
JSS_DEV void jss_st16<1>(uint16_t *p, const uint32_t (&o)[1]) { p[0] = (uint16_t)o[0]; }
template <>
JSS_DEV void jss_st16<2>(uint16_t *p, const uint32_t (&o)[2]) { *reinterpret_cast<uint32_t *>(p) = o[0] | (o[1] << 16); }
template <>
JSS_DEV void jss_st16<4>(uint16_t *p, const uint32_t (&o)[4]) {
    *reinterpret_cast<uint2 *>(p) = make_uint2(o[0] | (o[1] << 16), o[2] | (o[3] << 16));
}
template <>
JSS_DEV void jss_st16<8>(uint16_t *p, const uint32_t (&o)[8]) {
    uint4 v;
    v.x = o[0] | (o[1] << 16); v.y = o[2] | (o[3] << 16); v.z = o[4] | (o[5] << 16); v.w = o[6] | (o[7] << 16);
    *reinterpret_cast<uint4 *>(p) = v;
}

// a lane's legal / blocked bits inside the state block
template <int KJ>
JSS_DEV uint32_t jss_ld_bits(const int32_t *bits_region, int lane) {
    if (KJ == 8) return reinterpret_cast<const uint16_t *>(bits_region)[lane];
    return reinterpret_cast<const uint8_t *>(bits_region)[lane];
}
template <int KJ>
JSS_DEV void jss_st_bits(int32_t *bits_region, int lane, uint32_t lb) {
    if (KJ == 8) reinterpret_cast<uint16_t *>(bits_region)[lane] = (uint16_t)lb;
    else reinterpret_cast<uint8_t *>(bits_region)[lane] = (uint8_t)lb;
}

// ---- state block <-> registers -----------------------------------------------------
// Padding slots (job index >= J inside the last active lane, and whole lanes past the
// last job) hold todo == M, i.e. they behave like finished jobs everywhere.
template <int KJ>
JSS_DEV void env_derive_ops(const InstView &iv, EnvRegs<KJ> &s, int lane) {
    const int M = jss_M(iv);
    // lanes past the last job read row 0 (any in-bounds row: their todo == M selects JSS_OP_NONE anyway)
    const int row = (KJ * lane < jss_J(iv)) ? KJ * lane * M : 0;
#pragma unroll
    for (int i = 0; i < KJ; i++) {
        // unconditional load of a clamped index + select: no divergent branch around the table lookup
        const uint32_t o = iv.ops[row + i * M + min(s.todo[i], M - 1)];
        s.op[i] = (s.todo[i] < M) ? o : JSS_OP_NONE;
    }
}

template <int KJ>
JSS_DEV void env_clear_jobs(const InstView &iv, EnvRegs<KJ> &s) {
#pragma unroll
    for (int i = 0; i < KJ; i++) { s.todo[i] = jss_M(iv); s.tufco[i] = 0; s.idle_last[i] = 0; s.total_idle[i] = 0; s.col4[i] = 0; }
}

// The job records of the block (w0, w1, w2; jss_types.h) are decoded into the five EnvRegs arrays on load and
// encoded on store: everything between works on plain ints.
template <int KJ>
JSS_DEV void env_load_jobs(const int32_t *blk, int Jc, int lane, EnvRegs<KJ> &s) {
    int w0[KJ], w1[KJ];
    uint32_t w2[KJ];
    jss_ld<KJ>(blk + KJ * lane, w0);
    jss_ld<KJ>(blk + Jc + KJ * lane, w1);
    jss_ld16<KJ>(reinterpret_cast<const uint16_t *>(blk + 2 * Jc) + KJ * lane, w2);
#pragma unroll
    for (int i = 0; i < KJ; i++) {
        const uint32_t a = (uint32_t)w0[i], b = (uint32_t)w1[i];
        s.todo[i] = jss_job_todo(a);
        s.tufco[i] = jss_job_tufco(a);
        s.col4[i] = jss_job_col4(a);
        s.idle_last[i] = jss_job_idle_last(b);
        s.total_idle[i] = jss_job_total_idle(b, w2[i]);
    }
}

// a lane's legal / blocked bits and the env's header, behind the tuam words of the block
template <int KJ>
JSS_DEV void env_load_bits_hdr(const int32_t *tail, int Mc, int lane, EnvRegs<KJ> &s) {
    s.lb = jss_ld_bits<KJ>(tail + Mc, lane);
    const int4 h4 = *reinterpret_cast<const int4 *>(tail + Mc + jss_bits_words<KJ>());
    s.t = h4.x; s.flags = (uint32_t)h4.y; s.ep_steps = h4.z; s.ep_return = h4.w;
}

// `blk`: the env's state block (in global memory, or the step kernels' shared-memory copy)
template <int KJ>
JSS_DEV void env_load(const InstView &iv, const int32_t *blk, int lane, EnvRegs<KJ> &s) {
    const int Jc = iv.si->Jcap, Mc = iv.si->Mcap;   // geometry of the env's own instance
    if (KJ * lane < jss_J(iv)) env_load_jobs<KJ>(blk, Jc, lane, s);
    else env_clear_jobs<KJ>(iv, s);
    const int32_t *tail = blk + iv.si->tail;
    s.tuam = (lane < jss_M(iv)) ? tail[lane] : 0;
    env_load_bits_hdr<KJ>(tail, Mc, lane, s);
    env_derive_ops<KJ>(iv, s, lane);
}

// policy kernels read only what the rule looks at: bits + header always, todo for every
// rule (current op / remaining work / remaining ops), idle_last for FIFO
template <int KJ>
JSS_DEV void env_load_for_policy(const InstView &iv, const int32_t *blk, int lane, EnvRegs<KJ> &s, int rule) {
    const int Jc = iv.si->Jcap, Mc = iv.si->Mcap;
    env_clear_jobs<KJ>(iv, s);
    if (rule != JSS_RULE_RANDOM && KJ * lane < jss_J(iv)) {
        jss_ld<KJ>(blk + KJ * lane, s.todo);          // w0 (todo)
#pragma unroll
        for (int i = 0; i < KJ; i++) s.todo[i] = jss_job_todo((uint32_t)s.todo[i]);
        if (rule == JSS_RULE_FIFO) {                  // w1 (idle_last)
            jss_ld<KJ>(blk + Jc + KJ * lane, s.idle_last);
#pragma unroll
            for (int i = 0; i < KJ; i++) s.idle_last[i] = jss_job_idle_last((uint32_t)s.idle_last[i]);
        }
    }
    s.tuam = 0;
    env_load_bits_hdr<KJ>(blk + iv.si->tail, Mc, lane, s);
    if (rule != JSS_RULE_RANDOM) env_derive_ops<KJ>(iv, s, lane);
    else {
#pragma unroll
        for (int i = 0; i < KJ; i++) s.op[i] = JSS_OP_NONE;
    }
}

template <int KJ>
JSS_DEV void env_store_to(const InstView &iv, int32_t *blk, int lane, const EnvRegs<KJ> &s) {
    const int Jc = iv.si->Jcap, Mc = iv.si->Mcap;
    // lanes past the last job hold the "finished job" padding values (todo == M, the rest 0): the whole block is
    // defined, including the padding of the u16 region w2 up to a multiple of 16 bytes
    if (KJ * lane < ((Jc + 7) & ~7)) {
        int w0[KJ], w1[KJ];
        uint32_t w2[KJ];
#pragma unroll
        for (int i = 0; i < KJ; i++) {
            const JssJobWords r = jss_pack_job(s.todo[i], s.tufco[i], s.col4[i], s.idle_last[i], s.total_idle[i]);
            w0[i] = (int)r.w0; w1[i] = (int)r.w1; w2[i] = r.w2;
        }
        if (KJ * lane < Jc) {
            jss_st<KJ>(blk + KJ * lane, w0);
            jss_st<KJ>(blk + Jc + KJ * lane, w1);
        }
        jss_st16<KJ>(reinterpret_cast<uint16_t *>(blk + 2 * Jc) + KJ * lane, w2);
    }
    int32_t *tail = blk + iv.si->tail;
    if (lane < Mc) tail[lane] = (lane < jss_M(iv)) ? s.tuam : 0;
    jss_st_bits<KJ>(tail + Mc, lane, s.lb);
    if (lane == 0)
        *reinterpret_cast<int4 *>(tail + Mc + jss_bits_words<KJ>()) = make_int4(s.t, (int)s.flags, s.ep_steps, s.ep_return);
}

template <int KJ>
JSS_DEV void env_store(const InstView &iv, int32_t *blk, int lane, const EnvRegs<KJ> &s) {
    // all lanes must have finished env_load (every lane reads the shared header words)
    // before any lane overwrites the block: paths such as the auto-reset have no
    // collective between load and store
    __syncwarp();
    env_store_to<KJ>(iv, blk, lane, s);
}

// jss_env.py:145-181
template <int KJ>
JSS_DEV void env_reset_regs(const InstView &iv, EnvRegs<KJ> &s, int lane) {
    s.lb = 0u;
#pragma unroll
    for (int i = 0; i < KJ; i++) {
        const bool valid = KJ * lane + i < jss_J(iv);
        s.todo[i] = valid ? 0 : jss_M(iv);
        s.tufco[i] = 0; s.idle_last[i] = 0; s.total_idle[i] = 0; s.col4[i] = 0;
        if (valid) s.lb |= 1u << i;               // every job legal, no-op illegal (:160-161)
    }
    s.tuam = 0; s.t = 0; s.flags = 0u; s.ep_steps = 0; s.ep_return = 0;
    env_derive_ops<KJ>(iv, s, lane);
}

// ---- increase_time_step (jss_env.py:495-637); returns hole_planning ---------------
// TRACK: mark in s.dirty the job records the advance changes (the uniform step kernels' dirty-sector stores)
template <int KJ, bool TRACK = false>
JSS_DEV int env_advance(const InstView &iv, EnvRegs<KJ> &s, int lane) {
    // next event = smallest positive machine countdown (the sorted event list of
    // the reference always equals {t + tuam[m] : tuam[m] > 0}, appendix A.1)
    const int tuam_old = s.tuam;
    const int diff = (int)__reduce_min_sync(JSS_FULL, (unsigned)(tuam_old > 0 ? tuam_old : JSS_INF));
    const int gap = diff - tuam_old;                      // > 0 only for machines idle before the event
    const int hole = (int)__reduce_add_sync(JSS_FULL, (unsigned)((lane < jss_M(iv) && gap > 0) ? gap : 0));
    s.t += diff;
    const int M = jss_M(iv);
    const int row = (KJ * lane < jss_J(iv)) ? KJ * lane * M : 0;   // lanes past the last job: any in-bounds row
#pragma unroll
    for (int i = 0; i < KJ; i++) {
        // branch-free form of the reference's three cases (select instructions instead of divergent
        // branches): running (:529), running and finishing now (:550), waiting (:594); finished jobs
        // (todo == M) fall through unchanged
        const int was = s.tufco[i];
        const int left = was - diff;
        const bool running = was > 0;
        const bool finished = running && left <= 0;
        const bool waiting = !running && s.todo[i] < M;
        s.tufco[i] = left > 0 ? left : 0;                 // == max(0, was - diff); 0 stays 0
        const int slack = diff - was;                     // idle part of the step for a job finishing now
        const int idle = finished ? slack : (waiting ? diff : 0);
        s.total_idle[i] += idle;
        // w0 (tufco, and todo / col4 when finishing) of every running job, w1 (the idle times) of every waiting or
        // finishing one, and w2 only where total_idle >> 8 changed, i.e. where adding idle >= 0 carried out of the low
        // byte (then the low byte is now below idle): most advances leave it alone
        if (TRACK)
            s.dirty |= (running ? 1u << (JSS_DIRTY_W0 + i) : 0u) |
                       (waiting || finished ? 1u << (JSS_DIRTY_W1 + i) : 0u) |
                       ((s.total_idle[i] & 0xff) < idle ? 1u << (JSS_DIRTY_W2 + i) : 0u);
        s.idle_last[i] = finished ? slack : s.idle_last[i] + (waiting ? diff : 0);
        s.todo[i] += finished ? 1 : 0;
        {   // next op of a job that just finished one: unconditional clamped lookup + selects (no branch)
            const uint32_t o = iv.ops[row + i * M + min(s.todo[i], M - 1)];
            s.op[i] = finished ? ((s.todo[i] < M) ? o : JSS_OP_NONE) : s.op[i];
        }
        // real_obs[:,4] uses the PRE-decrement countdown of the next machine (:569-578)
        const int tq = __shfl_sync(JSS_FULL, tuam_old, (int)(jss_op_m(s.op[i]) & 31u));
        const int w = tq - diff;
        const int c4 = (s.op[i] != JSS_OP_NONE) ? (w > 0 ? w : 0) : iv.si->max_time_op;   // max_time_op encodes 1.0 (:586)
        s.col4[i] = finished ? c4 : s.col4[i];
    }
    s.tuam = gap < 0 ? -gap : 0;
    const uint32_t free_m = __ballot_sync(JSS_FULL, lane < jss_M(iv) && s.tuam == 0);
#pragma unroll
    for (int i = 0; i < KJ; i++)                          // legalisation (:616-634): free machine and not blocked
        s.lb |= (jss_bit(free_m, jss_op_m(s.op[i])) & ~(s.lb >> (jss_bs<KJ>() + i)) & 1u) << i;
    return hole;
}

// machines that have at least one legal job (== machine_legal of the reference)
template <int KJ>
JSS_DEV uint32_t env_machine_legal(const EnvRegs<KJ> &s) {
    uint32_t mine = 0u;
#pragma unroll
    for (int i = 0; i < KJ; i++) mine |= ((s.lb >> i) & 1u) << (jss_op_m(s.op[i]) & 31u);
    return __reduce_or_sync(JSS_FULL, mine);
}

// ---- _prioritization_non_final (jss_env.py:183-254) --------------------------------
template <int KJ>
JSS_DEV void env_prioritize(const InstView &iv, EnvRegs<KJ> &s, int lane) {
    uint32_t fin = 0u;                                    // my legal FINAL ops
    const int last = jss_M(iv) - 1;
#pragma unroll
    for (int i = 0; i < KJ; i++) fin |= (s.todo[i] == last ? 1u : 0u) << i;
    fin &= s.lb;
    if (!__any_sync(JSS_FULL, fin != 0u)) return;         // nothing can be de-legalised (the common case)
    uint32_t fin_m = 0u;                                  // machines wanted by a legal final op
#pragma unroll
    for (int i = 0; i < KJ; i++)
        if (fin & (1u << i)) fin_m |= 1u << (jss_op_m(s.op[i]) & 31u);
    fin_m = __reduce_or_sync(JSS_FULL, fin_m);
    const uint32_t free_m = __ballot_sync(JSS_FULL, lane < jss_M(iv) && s.tuam == 0);
    int cand_d[KJ];                                       // duration if legal non-final op whose NEXT machine is free
    const int row = KJ * lane * jss_M(iv);
#pragma unroll
    for (int i = 0; i < KJ; i++) {
        cand_d[i] = JSS_INF;
        if ((s.lb & (1u << i)) && !(fin & (1u << i))) {
            const uint32_t nxt = iv.ops[row + i * jss_M(iv) + s.todo[i] + 1];
            if (jss_bit(free_m, jss_op_m(nxt))) cand_d[i] = jss_op_d(s.op[i]);   // :234-239
        }
    }
    uint32_t kill = 0u;
    while (fin_m) {                                       // per machine with a legal final op
        const uint32_t m = (uint32_t)(__ffs((int)fin_m) - 1);
        fin_m &= fin_m - 1u;
        int mn = JSS_INF;
#pragma unroll
        for (int i = 0; i < KJ; i++)
            if (cand_d[i] != JSS_INF && jss_op_m(s.op[i]) == m) mn = min(mn, cand_d[i]);
        mn = (int)__reduce_min_sync(JSS_FULL, (unsigned)mn);   // min_non_final (:238)
        if (mn != JSS_INF) {
#pragma unroll
            for (int i = 0; i < KJ; i++)
                if ((fin & (1u << i)) && jss_op_m(s.op[i]) == m && jss_op_d(s.op[i]) > mn) kill |= 1u << i;  // :252
        }
    }
    s.lb &= ~kill;
}

// ---- _check_no_op (jss_env.py:256-401); returns legal_actions[J] -----------------
// `hz` is a 32-int per-warp shared scratch (aliases the observation staging area).
//
// Pass 1 visits the legal jobs one by one in ascending order, but nothing it decides depends on that order, so it runs
// once per legal machine (<= 3) with every lane taking its own jobs on the machine, one REDUX.MIN for the machine's
// shortest legal job:
// - it returns "not legal" iff some legal job ends before the next event, t + d < t + mn;
// - max_horizon_machine[m] ends as t + min(max_time_op, min d) over the legal jobs on m; pass 2 reads it only where
//   machine_legal[m], so elsewhere the table holds INT_MIN;
// - max_horizon, the largest value a running minimum takes at a visit, is t + the first legal job's d on some machine,
//   and can exceed H = the largest final minimum.  It only bounds pass 2's walks, and a walk step at a time >= H adds
//   nothing (that needs max_horizon_machine[m] > time for a legal m) while the time only grows: walking to H instead
//   gives the same machine_next in fewer steps.
// Pass 2 is order-free as well: machine_next only collects legal machines and only grows, so "it reached
// nb_machine_legal at some point" is "it equals machine_legal at the end", and each walk reads only the final table,
// the bound and its job's state.  Its early exits after a job slot whose walks cover every legal machine only save work
// (they end 43 % of the ta80 checks that reach pass 2 before the last slot, DESIGN.md §4).  Times are relative to t.
template <int KJ>
JSS_DEV bool env_check_no_op(const InstView &iv, const EnvRegs<KJ> &s, int lane, uint32_t ML, int nlegal,
                             int *hz) {
    const unsigned mn = __reduce_min_sync(JSS_FULL, (unsigned)(s.tuam > 0 ? s.tuam : JSS_INF));
    if (mn == (unsigned)JSS_INF || __popc(ML) > 3 || nlegal > 4) return false;   // gate :284-288
    const uint32_t lg = s.lb & jss_legal_mask<KJ>();
    const int mto = iv.si->max_time_op;                 // :300-302
    int maxh = 0;                                       // H - t
    int lm0 = -1, lm1 = -1, lm2 = -1, h0 = 0, h1 = 0, h2 = 0;   // the legal machines and their horizons - t
    uint32_t rest = ML;
#pragma unroll 1
    while (rest) {                                      // :305-321, warp-uniform
        const int m = __ffs((int)rest) - 1;
        rest &= rest - 1u;
        int d = JSS_INF;
#pragma unroll
        for (int i = 0; i < KJ; i++) {
            const bool on = ((lg >> i) & 1u) && (int)jss_op_m(s.op[i]) == m;
            // two spellings of one minimum: with these, ptxas (CUDA 12.9) keeps every kernel that inlines the check at
            // its launch bound without spills but jss_step_mixed_kernel<0, false> (DESIGN.md §4)
            d = KJ == 8 ? min(d, on ? jss_op_d(s.op[i]) : JSS_INF) : (on ? min(d, jss_op_d(s.op[i])) : d);
        }
        d = (int)__reduce_min_sync(JSS_FULL, (unsigned)d);
        if (d < (int)mn) return false;                  // :314-315
        d = min(mto, d);
        if (lm0 < 0) { lm0 = m; h0 = d; } else if (lm1 < 0) { lm1 = m; h1 = d; } else { lm2 = m; h2 = d; }
        maxh = max(maxh, d);
    }
    hz[lane] = (lane == lm0) ? h0 : (lane == lm1) ? h1 : (lane == lm2) ? h2 : (int)0x80000000;
    __syncwarp();
    const int last = jss_M(iv) - 1;
    // pass 2 (:324-401): jobs that are not legal now but may need a legal machine soon
    uint32_t want = 0u;
    const int row = KJ * lane * jss_M(iv);
#pragma unroll
    for (int i = 0; i < KJ; i++) {
        // countdown of the job's current machine (case 2, :374-377)
        const int tq = __shfl_sync(JSS_FULL, s.tuam, (int)(jss_op_m(s.op[i]) & 31u));
        if (!(s.lb & (1u << i)) && s.todo[i] < jss_M(iv)) {
            int ts, tm;
            if (s.tufco[i] > 0) { ts = s.todo[i] + 1; tm = s.tufco[i]; }            // case 1 (:327-337); a running
            else if (!(s.lb & ((1u << jss_bs<KJ>()) << i))) { ts = s.todo[i]; tm = tq; }   // last op walks nothing either way
            else { ts = jss_M(iv); tm = 0; }                                         // case 2 (:366-377) / blocked
            const uint16_t *o_ptr = iv.ops + row + i * jss_M(iv);
            while (ts < last && maxh > tm) {                                        // :340-342 / :380-382
                const uint32_t o = o_ptr[ts];
                if (hz[jss_op_m(o)] > tm) want |= 1u << jss_op_m(o);                // machine_next.add (:351 / :391)
                tm += jss_op_d(o);
                ts += 1;
            }
        }
        // the reference returns as soon as machine_next covers every legal machine (:357 / :395)
        if (i + 1 < KJ && ML != 0u && __reduce_or_sync(JSS_FULL, want) == ML) {
            __syncwarp();                               // hz aliases the obs staging buffer
            return true;
        }
    }
    want = __reduce_or_sync(JSS_FULL, want);
    __syncwarp();                                       // hz aliases the obs staging buffer
    return ML != 0u && want == ML;                      // len(machine_next) == nb_machine_legal
}

// Output bases of the emit helpers: the library's per-env buffers by default, the caller's trajectory buffers when a
// rollout records (then `env` is the trajectory slot k * N + env).
struct JssOut {
    float *obs;
    uint8_t *mask;
    int32_t *scalars;
};
JSS_DEV JssOut jss_out_default(const JssParams &p) { return JssOut{p.obs, p.mask, p.scalars}; }

// ---- dirty-sector stores of the uniform step kernels ---------------------------------------------
// The staged bytes (n16 16-byte chunks) leave by the warp's own 16-byte stores, but only the chunks in a 32-byte sector
// whose bit `sec` sets (absolute addresses: dst may start 16 bytes into a sector): a sector is written whole or not at
// all.  Bit k of word w of `sec`: sector 32 w + k counted from the one that holds dst[0].  NW words cover every sector
// and NIT rounds of 32 chunks every chunk of the largest n16 the caller passes.
template <int NW, int NIT>
JSS_DEV void jss_store_sectors(void *dst, const void *staged, int n16, const uint32_t (&sec)[NW], int lane) {
    // chunk k = lane + 32 it lies in sector 16 it + x: bit 16 (it & 1) + x of word it / 2 (or of the next word)
    const int x = ((int)((uintptr_t)dst & 31u) + 16 * lane) >> 5;
#pragma unroll
    for (int it = 0; it < NIT; it++) {
        const int k = lane + 32 * it, b = 16 * (it & 1) + x;
        const uint32_t m = b < 32 ? sec[it / 2] : sec[it / 2 + 1 < NW ? it / 2 + 1 : NW - 1];
        if (k < n16 && ((m >> (b & 31)) & 1u))
            reinterpret_cast<float4 *>(dst)[k] = reinterpret_cast<const float4 *>(staged)[k];
    }
    __syncwarp();
}

// The staged observation row: the sectors that hold a job whose row changed (env_dirty_rows).  This relies on real_obs
// holding, at the step's entry, the observation of the state block it loaded (jss_b200.h).
template <int KJ>
JSS_DEV void env_store_dirty_row(const EnvRegs<KJ> &s, float *dst, const float *staged, int n16, int lane) {
    constexpr int NW = (16 + 28 * 32 * KJ + 31) / 32 / 32 + 1;   // words for the largest row of the lane class
    const uint32_t rows = env_dirty_rows<KJ>(s);
    const int lead = (int)((uintptr_t)dst & 31u);
    const int r0 = lead + 28 * KJ * lane;                    // this lane's first row byte, from dst's first sector
    uint32_t loc = 0u;                                       // its jobs' sectors, from sector r0 >> 5 on
#pragma unroll
    for (int i = 0; i < KJ; i++) {
        const int a = ((r0 & 31) + 28 * i) >> 5, b = ((r0 & 31) + 28 * i + 27) >> 5;
        if (rows & (1u << i)) loc |= (2u << b) - (1u << a);
    }
    const uint64_t v = (uint64_t)loc << ((r0 >> 5) & 31);
    uint32_t sec[NW];
#pragma unroll
    for (int w = 0; w < NW; w++)
        sec[w] = __reduce_or_sync(JSS_FULL, (r0 >> 10) == w ? (uint32_t)v : (r0 >> 10) + 1 == w ? (uint32_t)(v >> 32) : 0u);
    jss_store_sectors<NW, (56 * KJ + 31) / 32>(dst, staged, n16, sec, lane);   // 7 J / 4 <= 56 KJ chunks
}

// 16-byte chunks of the lane class's largest state block (J = 32 KJ, M = 32: jss_block_geom)
template <int KJ>
JSS_DEV constexpr int jss_block16_max() { return (80 * KJ + 36 + 2 * jss_lane_slots(KJ)) / 4; }

// The staged state block: the sectors that hold a job record word s.dirty marks, every sector of the tail (tuam, the
// job bits and the header change at almost every step; its first sector may hold the end of w2) and the block's first
// sector.  The first and the last sector (in the tail) may be shared with the neighbouring blocks: storing this block's
// half of them always keeps such a sector whole in L2 when the neighbour does the same.  This relies on the block in
// HBM being, until the store, the block the step loaded.
template <int KJ>
JSS_DEV void env_store_dirty_block(const InstView &iv, const EnvRegs<KJ> &s, int32_t *dst, const int32_t *staged,
                                   int lane) {
    constexpr int N16 = jss_block16_max<KJ>(), NW = (16 * N16 + 16 + 1023) / 1024;
    const int lead = (int)((uintptr_t)dst & 31u);
    const int Jc = iv.si->Jcap;
    uint32_t loc[NW];                                        // this lane's changed sectors
#pragma unroll
    for (int w = 0; w < NW; w++) loc[w] = 0u;
    const auto mark = [&](int byte, uint32_t changed) {     // the sector of block byte `byte`, if `changed`
        const int g = (lead + byte) >> 5;
#pragma unroll
        for (int w = 0; w < NW; w++) loc[w] |= (changed != 0u && (g >> 5) == w) ? 1u << (g & 31) : 0u;
    };
    if (KJ * lane < jss_J(iv)) {
        // a lane's slice of w0 / w1 is 4 KJ bytes, of w2 2 KJ: each 16-byte piece of it lies in one sector
        constexpr int P = KJ > 4 ? KJ / 4 : 1, JP = KJ / P;
        constexpr uint32_t PM = (1u << JP) - 1u;
#pragma unroll
        for (int q = 0; q < P; q++) {
            mark(4 * (KJ * lane + JP * q), (s.dirty >> (JSS_DIRTY_W0 + JP * q)) & PM);
            mark(4 * (Jc + KJ * lane + JP * q), (s.dirty >> (JSS_DIRTY_W1 + JP * q)) & PM);
        }
        mark(8 * Jc + 2 * KJ * lane, (s.dirty >> JSS_DIRTY_W2) & jss_legal_mask<KJ>());
    }
    const int t0 = (lead + 4 * iv.si->tail) >> 5;            // the tail's first sector
    uint32_t sec[NW];
#pragma unroll
    for (int w = 0; w < NW; w++) {
        const int sh = t0 - 32 * w;
        sec[w] = __reduce_or_sync(JSS_FULL, loc[w]) | (w == 0 ? 1u : 0u) | (sh <= 0 ? ~0u : sh < 32 ? ~0u << sh : 0u);
    }
    jss_store_sectors<NW, (N16 + 31) / 32>(dst, staged, iv.si->block_words >> 2, sec, lane);
}

// ---- observation / mask / reward (jss_env.py:102-134, 483-493) ---------------------

template <int KJ, bool BULK = false, bool DIRTY = false>
JSS_DEV void env_emit_obs(const JssParams &p, const JssOut &out, const InstView &iv, const EnvRegs<KJ> &s, int env, int lane,
                          float *scratch, jss_saddr_t scratch_sa = jss_saddr_t(), void *st_dst = nullptr,
                          jss_saddr_t st_sa = jss_saddr_t(), uint32_t st_bytes = 0u) {
    if (KJ * lane < jss_J(iv)) {
        float v[KJ * 7];
#pragma unroll
        for (int i = 0; i < KJ; i++) {
            // total_perform_op_time_jobs == t - total_idle while the job is unfinished,
            // jobs_length[j] afterwards (every advance adds `difference` to exactly one of
            // the two counters until the job completes)
            const int len = iv.len[KJ * lane + i];        // unconditional (in-bounds) load + select
            const int perf = (s.todo[i] < jss_M(iv)) ? s.t - s.total_idle[i] : len;
            const JssInst &si = *iv.si;
            v[7 * i + 0] = (s.lb & (1u << i)) ? 1.0f : 0.0f;
            v[7 * i + 1] = jss_div((float)s.tufco[i], si.f_mto, si.r_mto);
            v[7 * i + 2] = jss_div((float)s.todo[i], si.f_M, si.r_M);
            v[7 * i + 3] = jss_div((float)perf, si.f_mtj, si.r_mtj);
            v[7 * i + 4] = jss_div((float)s.col4[i], si.f_mto, si.r_mto);
            v[7 * i + 5] = jss_div((float)s.idle_last[i], si.f_sop, si.r_sop);
            v[7 * i + 6] = jss_div((float)s.total_idle[i], si.f_sop, si.r_sop);
        }
        // stage the lane's 7*KJ floats (one contiguous, bank-conflict-free run per lane) ...
        float *mine = scratch + 7 * KJ * lane;
        if (KJ == 4 || KJ == 8) {
#pragma unroll
            for (int q = 0; q < 7 * KJ / 4; q++)
                reinterpret_cast<float4 *>(mine)[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
        } else if (KJ == 2) {
#pragma unroll
            for (int q = 0; q < 7; q++) reinterpret_cast<float2 *>(mine)[q] = make_float2(v[2 * q], v[2 * q + 1]);
        } else {
#pragma unroll
            for (int q = 0; q < 7; q++) mine[q] = v[q];
        }
    }
    float *dst = out.obs + (size_t)env * p.jobs_max * 7;
    const int n = jss_J(iv) * 7;
    if (BULK) {
        // ONE proxy fence covers both staged buffers (new state block + observation rows), then lane 0
        // hands them to the TMA engine: one bulk copy shared -> global each
        jss_fence_async_smem();          // make the generic-proxy writes visible to the async proxy
        __syncwarp();
        if (lane == 0) {
            if (st_bytes) jss_bulk_store(st_dst, st_sa, st_bytes);
            if ((n & 3) == 0 && (p.jobs_max & 3) == 0) jss_bulk_store(dst, scratch_sa, (uint32_t)n * 4u);
            jss_bulk_commit();           // ONE group for both copies (an empty group is legal)
        }
        if ((n & 3) == 0 && (p.jobs_max & 3) == 0)
            return;                      // the caller waits (wait_group.read) before reusing the staging buffers
    } else {
        __syncwarp();
        if (DIRTY && (n & 3) == 0 && (p.jobs_max & 3) == 0) {
            env_store_dirty_row<KJ>(s, dst, scratch, n >> 2, lane);
            return;
        }
    }
    // ... and stream the J*7 floats of the env out with fully coalesced stores
    int done_elems = 0;
    if ((p.jobs_max & 3) == 0) {
        const int n4 = n >> 2;
        for (int k = lane; k < n4; k += 32)
            reinterpret_cast<float4 *>(dst)[k] = reinterpret_cast<const float4 *>(scratch)[k];
        done_elems = n4 << 2;
    }
    for (int k = done_elems + lane; k < n; k += 32) dst[k] = scratch[k];
    __syncwarp();
}

template <int KJ>
JSS_DEV void env_emit_mask(const JssParams &p, const JssOut &out, const InstView &iv, const EnvRegs<KJ> &s, int env, int lane,
                           bool noop) {
    uint8_t *row = out.mask + (size_t)env * p.mask_stride;
    const int j0 = KJ * lane;
    if (KJ == 8) {
        if (j0 <= jss_J(iv)) {                            // 8 mask bytes per lane: two 4-bit spreads (rows are 8-byte aligned)
            uint32_t lo = ((s.lb & 15u) * 0x00204081u) & 0x01010101u, hi = (((s.lb >> 4) & 15u) * 0x00204081u) & 0x01010101u;
            const int d = jss_J(iv) - j0;                 // byte J is the no-op flag
            if (d < 4) lo |= (noop ? 1u : 0u) << (8 * d);
            else if (d < 8) hi |= (noop ? 1u : 0u) << (8 * (d - 4));
            *reinterpret_cast<uint2 *>(row + j0) = make_uint2(lo, hi);
        }
    } else if (j0 <= jss_J(iv)) {
        // spread the legal bits to bytes: bit i -> byte i
        // bit i -> byte i: the products of the set bits land on distinct positions (no carries)
        uint32_t w = ((s.lb & jss_legal_mask<KJ>()) * 0x00204081u) & 0x01010101u;
        if (jss_J(iv) - j0 < KJ) w |= (noop ? 1u : 0u) << (8 * (jss_J(iv) - j0));     // byte J is the no-op flag
        if (KJ == 4) *reinterpret_cast<uint32_t *>(row + j0) = w;
        else if (KJ == 2) *reinterpret_cast<uint16_t *>(row + j0) = (uint16_t)w;
        else row[j0] = (uint8_t)w;
    }
    if (jss_J(iv) == 32 * KJ && lane == 0) row[jss_J(iv)] = noop ? 1 : 0;   // no lane owns byte J
}

// reward / raw reward / time / (flags << 8 | done) of an env are ONE 16-byte record, so the
// per-step scalar outputs cost a single store (the API exposes them as strided arrays)
template <int KJ>
JSS_DEV void env_emit_scalars(const JssOut &out, const InstView &iv, const EnvRegs<KJ> &s, int env, int lane,
                              int raw_reward) {
    if (lane == 0) {
        const float r = jss_div((float)raw_reward, iv.si->f_mto, iv.si->r_mto);   // :483-493
        reinterpret_cast<int4 *>(out.scalars)[env] =
            make_int4(__float_as_int(r), raw_reward, s.t, (int)((s.flags << 8) | (s.flags & JSS_FLAG_DONE)));
    }
}

// episode bookkeeping when _is_done() turns true (jss_env.py:649-652)
template <int KJ>
JSS_DEV void env_episode_end(const JssParams &p, const EnvRegs<KJ> &s, int env, int lane) {
    if (lane == 0) {
        const int prev = p.episode_count[env];
        p.episode_count[env] = prev + 1;
        p.last_makespan[env] = s.t;
        p.last_return[env] = s.ep_return;
        int64_t *acc = p.acc + (size_t)env * 4;
        acc[0] += s.ep_steps;
        acc[1] += s.t;
        acc[2] += s.ep_return;
        const uint64_t mm = (uint64_t)acc[3];
        uint32_t mn = prev ? (uint32_t)(mm >> 32) : 0xffffffffu, mx = prev ? (uint32_t)mm : 0u;
        if ((uint32_t)s.t < mn) mn = (uint32_t)s.t;
        if ((uint32_t)s.t > mx) mx = (uint32_t)s.t;
        acc[3] = (int64_t)(((uint64_t)mn << 32) | mx);
    }
}

// a reset env's solution row (JSS_CREATE_RECORD_SOLUTION) holds -1 everywhere
JSS_DEV void env_clear_solution(const JssParams &p, int env, int lane) {
    if (p.solution) {
        int32_t *sol = p.solution + (size_t)env * p.jobs_max * p.machines_max;
        for (int k = lane; k < p.jobs_max * p.machines_max; k += 32) sol[k] = -1;
    }
}

// ---- step (jss_env.py:403-481) ---------------------------------------------------------
// Returns true if the env changed (outputs must be re-emitted).  BOOKKEEP = false (jss_lookahead's throw-away
// simulations) changes nothing but the registers: no solution entry, no episode statistics, no auto-reset.
// SOL_OUT (with BOOKKEEP = false: jss_sample_episodes_solution's replay) writes the allocated operation's start time
// into the caller's `sol_out`, which has the layout of p.solution, and nothing else.
template <int KJ, bool BOOKKEEP = true, bool TRACK = false, bool SOL_OUT = false>
JSS_DEV bool env_step(const JssParams &p, const InstView &iv, EnvRegs<KJ> &s, int env, int lane, int action,
                      int &raw_reward, int *hz, int32_t *sol_out = nullptr) {
    raw_reward = 0;
    if (action == JSS_ACTION_SKIP) return false;
    if (s.flags & JSS_FLAG_DONE) {
        if (BOOKKEEP && (p.create_flags & JSS_CREATE_AUTO_RESET)) {
            env_reset_regs<KJ>(iv, s, lane);
            if (TRACK) s.dirty = ~0u;
            env_clear_solution(p, env, lane);
            return true;
        }
        return false;  // frozen until reset
    }
    constexpr uint32_t LM = jss_legal_mask<KJ>();
    int holes = 0, gain = 0;
    const bool wait = (action == JSS_ACTION_ADVANCE || action == jss_J(iv));
    if (wait) {
        if (!__any_sync(JSS_FULL, s.tuam > 0)) { s.flags |= JSS_FLAG_ERROR; return false; }   // IndexError at :517
        if (action == jss_J(iv))                          // no-op (:419-428): legal -> blocked
            s.lb = ((s.lb & LM) << jss_bs<KJ>()) | (s.lb & (LM << jss_bs<KJ>()));
    } else {                                             // job allocation (:441-481)
        if (action < 0 || action > jss_J(iv)) { s.flags |= JSS_FLAG_ERROR; return false; }
        const int la = action / KJ, ia = action % KJ;
        const uint32_t opa = __shfl_sync(JSS_FULL, jss_sel<KJ>(s.op, ia), la);
        const uint32_t bits_a = __shfl_sync(JSS_FULL, s.lb, la);
        if (opa == JSS_OP_NONE || !((bits_a >> ia) & 1u)) { s.flags |= JSS_FLAG_ERROR; return false; }
        const uint32_t m_a = jss_op_m(opa);
        gain = jss_op_d(opa);
        s.tuam = ((uint32_t)lane == m_a) ? gain : s.tuam;            // :446
#pragma unroll
        for (int i = 0; i < KJ; i++) s.tufco[i] = (lane == la && i == ia) ? gain : s.tufco[i];   // :447
        if (TRACK && lane == la) s.dirty |= 1u << (JSS_DIRTY_W0 + ia);
        if (BOOKKEEP && p.solution && lane == la)                     // :454
            p.solution[((size_t)env * p.jobs_max + action) * p.machines_max + jss_sel<KJ>(s.todo, ia)] = s.t;
        if (SOL_OUT && lane == la)
            sol_out[((size_t)env * p.jobs_max + action) * p.machines_max + jss_sel<KJ>(s.todo, ia)] = s.t;
#pragma unroll
        for (int i = 0; i < KJ; i++)
            // every job waiting for machine m_a: no longer legal (:455-461), no longer
            // no-op-blocked (:464-467; illegal_actions[m][j] implies needed_machine[j]==m)
            if (jss_op_m(s.op[i]) == m_a) s.lb &= ~((((1u << jss_bs<KJ>()) | 1u)) << i);
    }
    // ONE inlined copy of the time advance serves the three callers: the raw hook (exactly one
    // advance), the no-op (:429-430, at least one) and the job branch (:469-470, zero or more)
    bool force = wait;
    uint32_t st;                                         // bit 0: some job is legal, bit 1: some event is pending
    for (;;) {
        st = __reduce_or_sync(JSS_FULL, ((s.lb & LM) != 0u ? 1u : 0u) | (s.tuam > 0 ? 2u : 0u));
        if (!(force || st == 2u)) break;                 // advance while nothing is legal and an event is pending
        holes += env_advance<KJ, TRACK>(iv, s, lane);
        force = false;
        if (action == JSS_ACTION_ADVANCE) { raw_reward = -holes; return true; }   // heuristics / _is_done do NOT run
    }
    if (action == jss_J(iv) && !(st & 1u))
        s.flags |= JSS_FLAG_ERROR;                       // the reference raises here (queue ran empty)
    raw_reward = gain - holes;
    env_prioritize<KJ>(iv, s, lane);                     // :432 / :471
    const uint32_t ML = env_machine_legal<KJ>(s);
    const int nlegal = (int)__reduce_add_sync(JSS_FULL, (unsigned)__popc(s.lb & LM));
    const bool noop = env_check_no_op<KJ>(iv, s, lane, ML, nlegal, hz);   // :433 / :472
    s.flags &= ~(JSS_FLAG_NOOP_LEGAL | JSS_FLAG_DONE);
    if (noop) s.flags |= JSS_FLAG_NOOP_LEGAL;
    s.ep_steps += 1;
    s.ep_return += raw_reward;
    if (nlegal == 0) {                                   // _is_done (:649)
        s.flags |= JSS_FLAG_DONE;
        if (BOOKKEEP) env_episode_end<KJ>(p, s, env, lane);
    }
    return true;
}

// ---- policies (JSSEnv/dispatching.py; README.md:58-60) ---------------------------------
template <int KJ, bool RANDOM_ONLY = false>
JSS_DEV int env_select_action(const InstView &iv, const EnvRegs<KJ> &s, int lane, int rule, int coin_mode,
                              uint32_t h, double cr_factor) {
    constexpr uint32_t LM = jss_legal_mask<KJ>();
    const uint32_t mine = (uint32_t)__popc(s.lb & LM);
    // inclusive prefix count of legal jobs over the lanes (ascending job index order)
    uint32_t incl = mine;
    int njobs;
    if (KJ == 1) {                                       // one job per lane: the prefix is a popcount of the ballot
        const uint32_t b = __ballot_sync(JSS_FULL, mine != 0u);
        incl = (uint32_t)__popc(b & ((2u << lane) - 1u));
        njobs = __popc(b);
    } else {
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const uint32_t o = __shfl_up_sync(JSS_FULL, incl, off);
            if (lane >= off) incl += o;
        }
        njobs = (int)__shfl_sync(JSS_FULL, incl, 31);
    }
    const bool noop = (s.flags & JSS_FLAG_NOOP_LEGAL) != 0u;
    if (s.flags & JSS_FLAG_DONE) return 0;               // ignored by step (auto-reset or frozen)
    if (njobs == 0) return noop ? jss_J(iv) : JSS_ACTION_SKIP;   // "only the no-op is legal" (e.g. :96-97)
    if (RANDOM_ONLY || rule == JSS_RULE_RANDOM) {
        // uniform over the set bits of action_mask, indexed in ascending action order
        const uint32_t r = jss_pick(h, (uint32_t)(njobs + (noop ? 1 : 0)));
        if ((int)r == njobs) return jss_J(iv);
        const uint32_t before = incl - mine;
        const bool own = r >= before && r < incl;
        int act = 0;
        uint32_t k = r - before;                         // k-th set slot of this lane (meaningful if `own`)
#pragma unroll
        for (int i = 0; i < KJ; i++) {
            const uint32_t bit = (s.lb >> i) & 1u;
            act = (bit && k == 0u) ? KJ * lane + i : act;
            k -= bit;
        }
        const uint32_t who = __ballot_sync(JSS_FULL, own);
        return __shfl_sync(JSS_FULL, act, __ffs((int)who) - 1);
    }
    int best;
    if (rule == JSS_RULE_CR) {                           // dispatching.py:365-408, float64 like Python
        double key = 1.0 / 0.0;
        int kj = 1 << 20;
#pragma unroll
        for (int i = 0; i < KJ; i++) {
            const int j = KJ * lane + i;
            if (s.lb & (1u << i)) {
                const double due = (double)iv.len[j] * cr_factor;                    // :357-360
                const int remaining = iv.rem[j * (jss_M(iv) + 1) + s.todo[i]];            // :387-388
                const double ratio = remaining > 0 ? (due - (double)s.t) / (double)remaining : 1.0 / 0.0;
                if (ratio < key) { key = ratio; kj = j; }                            // strict <, first index wins
            }
        }
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) {
            const double ok = __shfl_xor_sync(JSS_FULL, key, off);
            const int oj = __shfl_xor_sync(JSS_FULL, kj, off);
            if (ok < key || (ok == key && oj < kj)) { key = ok; kj = oj; }
        }
        best = kj;
    } else {
        // integer keys; composite (key << 8 | tie) so one REDUX picks value and first index
        const bool minimise = (rule == JSS_RULE_SPT || rule == JSS_RULE_LWR || rule == JSS_RULE_LOR);
        uint32_t comp = minimise ? 0xffffffffu : 0u;
#pragma unroll
        for (int i = 0; i < KJ; i++) {
            const int j = KJ * lane + i;
            if (s.lb & (1u << i)) {
                uint32_t key;
                if (rule == JSS_RULE_SPT) key = (uint32_t)jss_op_d(s.op[i]);                    // :105-108
                else if (rule == JSS_RULE_FIFO) key = (uint32_t)s.idle_last[i];                 // :146-148
                else if (rule == JSS_RULE_MWR || rule == JSS_RULE_LWR)
                    key = iv.rem[j * (jss_M(iv) + 1) + s.todo[i]];                                   // :188-191 / :231-234
                else key = (uint32_t)(jss_M(iv) - s.todo[i]);                                        // :273 / :314
                const uint32_t c = minimise ? ((key << 8) | (uint32_t)j) : ((key << 8) | (uint32_t)(255 - j));
                comp = minimise ? min(comp, c) : max(comp, c);
            }
        }
        comp = minimise ? __reduce_min_sync(JSS_FULL, comp) : __reduce_max_sync(JSS_FULL, comp);
        best = minimise ? (int)(comp & 255u) : 255 - (int)(comp & 255u);
    }
    if (noop && coin_mode == JSS_COIN_DEVICE && h < JSS_COIN_THRESHOLD) return jss_J(iv);   // e.g. :113-114
    return best;
}

// ---- masked categorical draw from policy logits (jss_step_logits, jss_b200.h) ----------------------------------
#define JSS_F32_INF __int_as_float(0x7f800000)
#define JSS_F32_NAN __int_as_float(0x7fffffff)
// unsigned key with the order of the floats (NaN aside), so one REDUX.MAX finds a warp maximum
JSS_DEV uint32_t jss_f32_key(float x) {
    const uint32_t b = (uint32_t)__float_as_int(x);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
JSS_DEV float jss_key_f32(uint32_t k) { return __int_as_float((int)((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k)); }
// The draw's log / exp: the MUFU approximations (a few ulp, absolute error 2^-21.4 near 1) are well inside what a
// sampler needs, and they are shorter: a build with libm's logf / expf spilled 28 bytes in the uniform 1-job-per-lane
// kernel at 64 registers, this one spills nothing.  log1pf stays, for -log u close to 0.  The host emulation uses libm.
#ifndef JSS_EMU
JSS_DEV float jss_fast_log(float x) { return __logf(x); }
JSS_DEV float jss_fast_exp(float x) { return __expf(x); }
#else
JSS_DEV float jss_fast_log(float x) { return logf(x); }
JSS_DEV float jss_fast_exp(float x) { return expf(x); }
#endif

// Gumbel noise g = -log(-log u) of u = ((bits >> 8) + 0.5) * 2^-24.  fp32 cannot hold every u close to 1
// (u = 1 - 2^-25 would round to 1 and give g = +inf), so the upper half works with 1 - u, which it holds exactly.
JSS_DEV float jss_gumbel(uint32_t bits) {
    const uint32_t k = bits >> 8;
    const float e = k < (1u << 23) ? -jss_fast_log(((float)k + 0.5f) * 0x1p-24f)
                                   : -log1pf(-(((float)((1u << 24) - 1u - k) + 0.5f) * 0x1p-24f));
    return -jss_fast_log(e);
}

// Gumbel-max over the actions legal in the env's current state: a = argmax((logit[a] - mx) + g[a]) in fp32 (lowest
// index on ties), mx the largest legal logit, g[a] from jss_hash_env(h, a) with h = jss_hash3(seed, global env id,
// step_index), and log_prob = (logit[a] - mx) - log(sum exp(legal logit - mx)).  The key is formed on the max-
// subtracted logit: on logit[a] itself, the noise would drown in the ulp of a large logit (every g lost at 1e30, ties
// to the lowest index), and the draw would stop following the log_prob it reports.  `row` holds the env's logits,
// columns 0..J; only legal columns are read.  Writes what the call reports to act / logp and returns the action to
// apply: the drawn one, 0 for a done env, or, for bad logits, an out-of-range action, so that env_step sets the
// sticky error bit and changes nothing else.
template <int KJ>
JSS_DEV int env_sample_logits(const InstView &iv, const EnvRegs<KJ> &s, int lane, const float *row, uint32_t h,
                              int &act, float &logp) {
    constexpr uint32_t LM = jss_legal_mask<KJ>();
    const uint32_t flags = jss_uniform(s.flags);
    const int J = jss_J(iv);
    const bool noop = (flags & JSS_FLAG_NOOP_LEGAL) != 0u;
    act = 0;
    logp = 0.0f;
    if (flags & JSS_FLAG_DONE) return 0;                 // reset or frozen by env_step, as with any action
    if (!__any_sync(JSS_FULL, (s.lb & LM) != 0u)) {      // only the no-op is legal (its logit is not read)
        act = noop ? J : JSS_ACTION_SKIP;
        logp = noop ? 0.0f : JSS_F32_NAN;
        return act;
    }
    // candidates: this lane's legal jobs in ascending order, then (lane 0) the legal no-op
    bool bad = false;                                    // a legal logit is NaN or +inf
    uint32_t xkey = 0u;                                  // 0: below every candidate's key
#pragma unroll
    for (int i = 0; i <= KJ; i++) {
        const bool cand = i < KJ ? ((s.lb >> i) & 1u) != 0u : (lane == 0 && noop);
        if (cand) {
            const float x = row[i < KJ ? KJ * lane + i : J];
            bad = bad || !(x < JSS_F32_INF);
            xkey = max(xkey, jss_f32_key(x));
        }
    }
    const float mx = jss_key_f32(__reduce_max_sync(JSS_FULL, xkey));
    if (__any_sync(JSS_FULL, bad) || mx == -JSS_F32_INF) {   // bad logits, or every legal logit is -inf
        act = JSS_ACTION_SKIP;
        logp = JSS_F32_NAN;
        return JSS_INF;
    }
    // the keys and the exponentials in one pass over d = x - mx (-inf where x - mx overflows: never drawn)
    uint32_t skey = 0u;                                  // 0: below every candidate's key
    int sidx = 1 << 20;
    float sum = 0.0f;
#pragma unroll
    for (int i = 0; i <= KJ; i++) {
        const bool cand = i < KJ ? ((s.lb >> i) & 1u) != 0u : (lane == 0 && noop);
        const int j = i < KJ ? KJ * lane + i : J;
        if (cand) {
            const float d = row[j] - mx;
            const uint32_t k = jss_f32_key(d + jss_gumbel(jss_hash_env(h, (uint64_t)j)));
            if (k > skey) { skey = k; sidx = j; }
            sum += jss_fast_exp(d);
        }
    }
    const uint32_t best = __reduce_max_sync(JSS_FULL, skey);
    act = (int)__reduce_min_sync(JSS_FULL, (unsigned)(skey == best ? sidx : 1 << 20));
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) sum += __shfl_xor_sync(JSS_FULL, sum, off);   // the same sum in every lane
    logp = (row[act] - mx) - jss_fast_log(sum);
    return act;
}

// The legal action with the largest value, ties to the lowest index, the values compared as IEEE floats (-0 and +0
// tie).  Candidates: this lane's legal jobs in ascending order, then (lane 0, if `noop`) the no-op J; `value(i, j)`
// gives candidate j's value, i its slot in the lane (KJ for the no-op), and is called for candidates only.  Returns
// false, leaving g alone, for a bad set: a candidate NaN or +inf, or every candidate -inf.  At least one job must be
// legal.
template <int KJ, typename Value>
JSS_DEV bool env_legal_argmax(const EnvRegs<KJ> &s, int lane, int J, bool noop, const Value &value, int &g) {
    bool bad = false;                                    // a candidate's value is NaN or +inf
    uint32_t key = 0u;                                   // 0: below every candidate's key
    int gidx = 1 << 20;
#pragma unroll
    for (int i = 0; i <= KJ; i++) {
        const bool cand = i < KJ ? ((s.lb >> i) & 1u) != 0u : (lane == 0 && noop);
        const int j = i < KJ ? KJ * lane + i : J;
        if (cand) {
            const float x = value(i, j);
            bad = bad || !(x < JSS_F32_INF);
            const uint32_t k = jss_f32_key(x + 0.0f);    // -0 + 0 = +0: jss_f32_key alone orders -0 below +0
            if (k > key) { key = k; gidx = j; }
        }
    }
    const uint32_t best = __reduce_max_sync(JSS_FULL, key);
    if (__any_sync(JSS_FULL, bad) || jss_key_f32(best) == -JSS_F32_INF) return false;
    g = (int)__reduce_min_sync(JSS_FULL, (unsigned)(key == best ? gidx : 1 << 20));
    return true;
}

// Epsilon-greedy decode of a row of scores (logits or Q-values; jss_step_greedy).  The greedy action g is the legal
// action with the largest score, ties to the lowest index, the scores compared as IEEE floats (-0 and +0 tie).  With
// T = explore_t (0 .. 2^32, set on the host), the env explores iff jss_hash_env(h, 0) < T, and then takes the
// masked-uniform pick of JSS_RULE_RANDOM drawn with jss_hash_env(h, 1): a separate hash, so that a small T does not
// bias the pick to the lowest legal actions.  log_prob = log((a == g ? 1 - e : 0) + e / n), e = T * 2^-32, n = the
// legal actions (the legal no-op included); exactly 0 for T = 0.  `row`, the special cases, the bad-row test (before
// the coin, so it never depends on the RNG) and the return value are those of env_sample_logits.
template <int KJ>
JSS_DEV int env_greedy_scores(const InstView &iv, const EnvRegs<KJ> &s, int lane, const float *row, uint32_t h,
                              uint64_t explore_t, int &act, float &logp) {
    constexpr uint32_t LM = jss_legal_mask<KJ>();
    const uint32_t flags = jss_uniform(s.flags);
    const int J = jss_J(iv);
    const bool noop = (flags & JSS_FLAG_NOOP_LEGAL) != 0u;
    act = 0;
    logp = 0.0f;
    if (flags & JSS_FLAG_DONE) return 0;                 // reset or frozen by env_step, as with any action
    if (!__any_sync(JSS_FULL, (s.lb & LM) != 0u)) {      // only the no-op is legal (its score is not read)
        act = noop ? J : JSS_ACTION_SKIP;
        logp = noop ? 0.0f : JSS_F32_NAN;
        return act;
    }
    int g;
    if (!env_legal_argmax<KJ>(s, lane, J, noop, [&](int, int j) { return row[j]; }, g)) {   // bad, or all -inf
        act = JSS_ACTION_SKIP;
        logp = JSS_F32_NAN;
        return JSS_INF;
    }
    act = g;
    if (explore_t != 0u) {                               // launch-uniform: a greedy launch neither counts nor draws
        // the pick is env_select_action's JSS_RULE_RANDOM branch itself (its done / nothing-legal cases do not apply
        // here).  n is its own REDUX.ADD: sharing the pick's prefix count means factoring it out of env_select_action,
        // which changes the code of the masked-uniform step kernels (SAMPLE = 1).
        if ((uint64_t)jss_hash_env(h, 0) < explore_t)
            act = env_select_action<KJ, true>(iv, s, lane, JSS_RULE_RANDOM, JSS_COIN_NEVER, jss_hash_env(h, 1), 0.0);
        const float n = (float)(__reduce_add_sync(JSS_FULL, (unsigned)__popc(s.lb & LM)) + (noop ? 1u : 0u));
        const float e = (float)explore_t * 0x1p-32f;
        // a == g: log(1 - y), y = e (n - 1) / n, through log1p while y is small (log would round 1 - y first); the
        // 0 - y keeps y = 0 (n = 1) at log_prob +0
        const float y = e * (n - 1.0f) / n;
        logp = act != g ? logf(e / n) : y < 0.5f ? log1pf(0.0f - y) : logf((1.0f - e) + e / n);
    }
    return act;
}

// ---- caller's priority table (jss_rollout_priority) -------------------------------------------------------------
// Env `env`'s part of a caller's table, hoisted out of the job loops, and its entry for operation k of job j
JSS_DEV const float *jss_table_row(const JssTable &t, int env) { return t.p + (int64_t)env * t.ld_env; }
JSS_DEV float jss_table_at(const JssTable &t, const float *row, int j, int k) {
    return row[(int64_t)j * t.ld_job + (int64_t)k * t.ld_op];
}

// Env `env`'s next action under its priority table (a.table): the legal job whose current operation has the largest
// priority, by env_legal_argmax without the no-op; the no-op only when no job is legal and it is.  Each lane loads the
// entries of its own legal jobs' current operations, nothing else.  Returns JSS_INF for bad priorities and
// JSS_ACTION_SKIP when nothing is legal (an imported state).
template <int KJ>
JSS_DEV int env_priority_action(const JssLaunch &a, const InstView &iv, const EnvRegs<KJ> &s, int env, int lane) {
    constexpr uint32_t LM = jss_legal_mask<KJ>();
    if (!__any_sync(JSS_FULL, (s.lb & LM) != 0u))
        return (s.flags & JSS_FLAG_NOOP_LEGAL) ? jss_J(iv) : JSS_ACTION_SKIP;
    const float *row = jss_table_row(a.table, env);
    int g = JSS_INF;
    env_legal_argmax<KJ>(s, lane, jss_J(iv), false, [&](int i, int j) {
        return jss_table_at(a.table, row, j, jss_sel<KJ>(s.todo, i));
    }, g);
    return g;
}

// The entropy of one decision's softmax over the legal jobs, from each owned slot's d_i = x_i - mx and e_i =
// jss_fast_exp(d_i) (e_i = 0 for a slot that is not legal), S = sum e_i and ls = jss_fast_log(S) as the decision source
// formed them: H = ls - T / S, T = sum over e_i > 0 of e_i d_i, summed in S's order (each lane's slots ascending, then
// the same butterfly).  A term with e_i = 0 (a legal job at -inf, or an exponential that underflows) adds nothing, so
// 0 * -inf never makes a NaN, and a decision with one job of nonzero probability gives exactly +0.  The one helper both
// decision sources call, so that an order's entropy and a draw's agree bit for bit.
template <int KJ>
JSS_DEV float jss_softmax_entropy(const float (&d)[KJ], const float (&e)[KJ], float sum, float ls) {
    float t = 0.0f;
#pragma unroll
    for (int i = 0; i < KJ; i++)
        if (e[i] > 0.0f) t += e[i] * d[i];
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) t += __shfl_xor_sync(JSS_FULL, t, off);
    return ls - t / sum;
}

// What a decision source reports besides the log-probability when asked for the entropy: H of the decision
// (jss_softmax_entropy; 0 for a forced no-op) and each owned slot's p_i (lp_i + H), the negated gradient term of H
// with respect to x_i (0 where p_i = 0, so lp_i = -inf makes no NaN).
template <int KJ>
struct JssEnt {
    float h;
    float q[KJ];
};
template <int KJ>
JSS_DEV void jss_ent_clear(JssEnt<KJ> *ent) {
    ent->h = 0.0f;
#pragma unroll
    for (int i = 0; i < KJ; i++) ent->q[i] = 0.0f;
}

// Env `env`'s next decision under its logit table (jss_rollout_priority_sample; the table as in env_priority_action):
// the Gumbel-max draw of env_sample_logits over the legal jobs, x_j = the entry of job j's current operation.  It
// equals env_sample_logits on the row x with the no-op column at -inf, bit for bit: the same keys and reductions, and
// the sum of exponentials in the same order (the no-op's exp(-inf) adds +0).  Kept apart from env_sample_logits, which
// reads a row in shared memory and puts the no-op among the candidates: a version shared with it would branch on both.
// Writes logp = x_a - logsumexp(x) and each owned slot's p_i = softmax(x)_j (0 for a job that is not legal).  Returns
// the drawn job; the no-op, logp and p left 0, when no job is legal and it is; JSS_INF for a bad table (the bad-row
// rule of env_sample_logits); JSS_ACTION_SKIP when nothing is legal (an imported state).
// ENT: also the decision's entropy and gradient terms into *ent (JssEnt; left 0 where logp is left 0).
template <int KJ, bool ENT = false>
JSS_DEV int env_priority_sample_action(const JssLaunch &a, const InstView &iv, const EnvRegs<KJ> &s, int env, int lane,
                                       uint32_t h, float &logp, float (&pr)[KJ], JssEnt<KJ> *ent = nullptr) {
    constexpr uint32_t LM = jss_legal_mask<KJ>();
    logp = 0.0f;
#pragma unroll
    for (int i = 0; i < KJ; i++) pr[i] = 0.0f;
    if constexpr (ENT) jss_ent_clear<KJ>(ent);
    if (!__any_sync(JSS_FULL, (s.lb & LM) != 0u))
        return (s.flags & JSS_FLAG_NOOP_LEGAL) ? jss_J(iv) : JSS_ACTION_SKIP;
    const float *row = jss_table_row(a.table, env);
    bool bad = false;                                    // a legal entry is NaN or +inf
    uint32_t xkey = 0u;                                  // 0: below every candidate's key
    float x[KJ];
#pragma unroll
    for (int i = 0; i < KJ; i++) {
        x[i] = 0.0f;
        if ((s.lb >> i) & 1u) {
            x[i] = jss_table_at(a.table, row, KJ * lane + i, s.todo[i]);
            bad = bad || !(x[i] < JSS_F32_INF);
            xkey = max(xkey, jss_f32_key(x[i]));
        }
    }
    const float mx = jss_key_f32(__reduce_max_sync(JSS_FULL, xkey));
    if (__any_sync(JSS_FULL, bad) || mx == -JSS_F32_INF) return JSS_INF;   // bad entries, or every legal one -inf
    uint32_t skey = 0u;                                  // 0: below every candidate's key
    int sidx = 1 << 20;
    float sd = 0.0f, sum = 0.0f;                         // sd: x - mx of this lane's best candidate
#pragma unroll
    for (int i = 0; i < KJ; i++) {
        if ((s.lb >> i) & 1u) {
            const int j = KJ * lane + i;
            const float d = x[i] - mx;
            const uint32_t k = jss_f32_key(d + jss_gumbel(jss_hash_env(h, (uint64_t)j)));
            if (k > skey) { skey = k; sidx = j; sd = d; }
            pr[i] = jss_fast_exp(d);
            sum += pr[i];
            if constexpr (ENT) x[i] = d;
        }
    }
    const uint32_t best = __reduce_max_sync(JSS_FULL, skey);
    const int act = (int)__reduce_min_sync(JSS_FULL, (unsigned)(skey == best ? sidx : 1 << 20));
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) sum += __shfl_xor_sync(JSS_FULL, sum, off);   // the same sum in every lane
    const float da = __shfl_sync(JSS_FULL, sd, act / KJ);   // the drawn job's lane holds it as its best candidate
    logp = da - jss_fast_log(sum);
    if constexpr (ENT) ent->h = jss_softmax_entropy<KJ>(x, pr, sum, jss_fast_log(sum));   // pr: still e_i
    const float inv = 1.0f / sum;
#pragma unroll
    for (int i = 0; i < KJ; i++) pr[i] *= inv;
    if constexpr (ENT) {
        const float ls = jss_fast_log(sum);
#pragma unroll
        for (int i = 0; i < KJ; i++) ent->q[i] = pr[i] > 0.0f ? pr[i] * ((x[i] - ls) + ent->h) : 0.0f;
    }
    return act;
}

// ---- canonical export / import (snapshot & restore; host attribute views) -------------
template <int KJ>
JSS_DEV void env_export(const JssParams &p, const InstView &iv, const EnvRegs<KJ> &s, int env, int lane) {
    const size_t jb = (size_t)env * p.jobs_max;
#pragma unroll
    for (int i = 0; i < KJ; i++) {
        const int j = KJ * lane + i;
        if (j < jss_J(iv)) {
            p.x_todo[jb + j] = s.todo[i]; p.x_tufco[jb + j] = s.tufco[i];
            p.x_idle_last[jb + j] = s.idle_last[i]; p.x_total_idle[jb + j] = s.total_idle[i];
            p.x_col4[jb + j] = s.col4[i];
            p.x_legal[jb + j] = (uint8_t)((s.lb >> i) & 1u);
            p.x_blocked[jb + j] = (uint8_t)((s.lb >> (jss_bs<KJ>() + i)) & 1u);
        }
    }
    if (lane < jss_M(iv)) p.x_tuam[(size_t)env * p.machines_max + lane] = s.tuam;
    if (lane == 0) {
        p.scalars[4 * (size_t)env + 2] = s.t;
        p.scalars[4 * (size_t)env + 3] = (int32_t)((s.flags << 8) | (s.flags & JSS_FLAG_DONE));
    }
}

// The job records keep todo in [0, M], tufco and col4 in [0, 2047], idle_last and total_idle in [0, 2^24)
// (jss_types.h).  An imported value outside its range is clamped into it and the env gets the sticky error bit.
static_assert(JSS_MAX_MACHINES <= (int)JSS_PACK_TODO_MASK && JSS_MAX_DURATION <= (int)JSS_PACK_DUR_MASK,
              "the job record must hold every todo and duration the kernels accept");
template <int KJ>
JSS_DEV void env_import(const JssParams &p, const InstView &iv, EnvRegs<KJ> &s, int env, int lane) {
    const size_t jb = (size_t)env * p.jobs_max;
    s.lb = 0u;
    bool bad = false;
    const auto take = [&bad](int v, int hi) { bad = bad || v < 0 || v > hi; return min(max(v, 0), hi); };
#pragma unroll
    for (int i = 0; i < KJ; i++) {
        const int j = KJ * lane + i;
        const bool valid = j < jss_J(iv);
        s.todo[i] = valid ? take(p.x_todo[jb + j], jss_M(iv)) : jss_M(iv);
        s.tufco[i] = valid ? take(p.x_tufco[jb + j], (int)JSS_PACK_DUR_MASK) : 0;
        s.idle_last[i] = valid ? take(p.x_idle_last[jb + j], JSS_PACK_IDLE_MAX) : 0;
        s.total_idle[i] = valid ? take(p.x_total_idle[jb + j], JSS_PACK_IDLE_MAX) : 0;
        s.col4[i] = valid ? take(p.x_col4[jb + j], (int)JSS_PACK_DUR_MASK) : 0;
        if (valid && p.x_legal[jb + j] != 0) s.lb |= 1u << i;
        if (valid && p.x_blocked[jb + j] != 0) s.lb |= (1u << jss_bs<KJ>()) << i;
    }
    s.tuam = lane < jss_M(iv) ? p.x_tuam[(size_t)env * p.machines_max + lane] : 0;
    s.t = p.scalars[4 * (size_t)env + 2];
    s.flags = (uint32_t)p.scalars[4 * (size_t)env + 3] >> 8;
    if (__any_sync(JSS_FULL, bad)) s.flags |= JSS_FLAG_ERROR;
    env_derive_ops<KJ>(iv, s, lane);
}

// ---- packed observation row (host-buffer path) ---------------------------------------------------------
// One job record per job (jss_types.h, 10 bytes), with the legal bit in w0.  Column 3 (total_perform) is derivable
// on the host from total_idle, todo, t and jobs_length.  jss_host_expand_obs() turns a row back into the exact
// real_obs floats.
template <int KJ>
JSS_DEV void env_pack(const JssLaunch &a, const InstView &iv, const EnvRegs<KJ> &s, int env, int lane, float *scratch) {
    uint16_t *st = reinterpret_cast<uint16_t *>(scratch);
    if (KJ * lane < jss_J(iv)) {
#pragma unroll
        for (int i = 0; i < KJ; i++) {
            const JssJobWords w = jss_pack_job(s.todo[i], s.tufco[i], s.col4[i], s.idle_last[i], s.total_idle[i]);
            const uint32_t w0 = w.w0 | (((s.lb >> i) & 1u) << JSS_PACK_LEGAL_SHIFT);
            uint16_t *r = st + 5 * (KJ * lane + i);   // 2-byte aligned: stored as five u16
            r[0] = (uint16_t)w0; r[1] = (uint16_t)(w0 >> 16);
            r[2] = (uint16_t)w.w1; r[3] = (uint16_t)(w.w1 >> 16);
            r[4] = (uint16_t)w.w2;
        }
    }
    __syncwarp();
    uint4 *dst = reinterpret_cast<uint4 *>(a.wire + (size_t)env * a.wire_stride);
    const int n16 = (jss_J(iv) * 10 + 15) >> 4;
    for (int k = lane; k < n16; k += 32) dst[k] = reinterpret_cast<const uint4 *>(scratch)[k];
    __syncwarp();
}

// ---- CTA-level driver -----------------------------------------------------------------------
struct JssSmemLayout {
    // byte offsets from the start of dynamic shared memory, precomputed on the host so the kernels derive every
    // pointer with one add (each region 16-byte aligned): [JssInst][ops u16][len i32][rem u16][per-warp regions]
    int32_t off_len, off_rem, off_warp0, pad0_;
    int32_t warp_stride;    // bytes per warp region
    int32_t scratch_words;  // observation staging (7 floats per job slot), >= 32 words
    int32_t off_scratch;    // step kernels: [mbarrier 16 B][state-in block][scratch][state-out block]; else 0
    int32_t off_logits;     // step kernels that take a row: [logits row, J + 1 floats] behind state-out; else 0
};
static_assert(sizeof(JssParams) == 248 && sizeof(JssLaunch) == 496 && sizeof(JssSmemLayout) == 32 &&
              sizeof(JssTile) == 16 && sizeof(JssCtaRange) == 32,
              "ptxas allocates the kernels' registers by the parameter offsets (JssParams::pad0_): measure a change");
// the same for the fields of JssLaunch that the fused step kernels read
static_assert(offsetof(JssLaunch, tile_begin) == 0 && offsetof(JssLaunch, tile_end) == 4 &&
              offsetof(JssLaunch, rule) == 12 && offsetof(JssLaunch, coin_mode) == 16 &&
              offsetof(JssLaunch, explore_t) == 32 && offsetof(JssLaunch, hash_key) == 48 &&
              offsetof(JssLaunch, stage) == 52 && offsetof(JssLaunch, cr_factor) == 56 &&
              offsetof(JssLaunch, actions) == 64 && offsetof(JssLaunch, actions_out) == 72 &&
              offsetof(JssLaunch, traj_obs) == 88 && offsetof(JssLaunch, traj_mask) == 96 &&
              offsetof(JssLaunch, traj_scalars) == 104 && offsetof(JssLaunch, uni) == 132 &&
              offsetof(JssLaunch, rows) == 216 && offsetof(JssLaunch, log_prob_out) == 224 &&
              offsetof(JssLaunch, rows_ld) == 232,
              "ptxas allocates the step kernels' registers by the parameter offsets: measure a change");

struct JssCtaSmem {         // the CTA-shared part
    JssInst *si;
    uint16_t *ops;
    int32_t *len;
    uint16_t *rem;
};
JSS_DEV void jss_cta_carve(const JssSmemLayout &sl, char *sm, JssCtaSmem &c, InstView &iv) {
    c.si = reinterpret_cast<JssInst *>(sm);
    c.ops = reinterpret_cast<uint16_t *>(sm + sizeof(JssInst));
    c.len = reinterpret_cast<int32_t *>(sm + sl.off_len);
    c.rem = reinterpret_cast<uint16_t *>(sm + sl.off_rem);
    iv.ops = c.ops; iv.len = c.len; iv.rem = c.rem; iv.si = c.si; iv.staged = true; iv.Ju = iv.Mu = 0;
}

// refresh the uniform register copies of J / M from the staged instance (one packed shuffle)
JSS_DEV void jss_iv_shape(InstView &iv) {
    const uint32_t jm = jss_uniform((uint32_t)iv.si->J | ((uint32_t)iv.si->M << 16));
    iv.Ju = (int)(jm & 0xffffu); iv.Mu = (int)(jm >> 16);
}

#define JSS_STAGE_OPS 1     // ops + jobs_length
#define JSS_STAGE_REM 2     // suffix sums (rules MWR / LWR / CR)
#define JSS_STAGE_ALL 3

JSS_DEV void jss_stage_instance(const JssParams &p, const JssInst &d, const JssCtaSmem &c, int what) {
    const int tid = threadIdx.x, nt = blockDim.x;
    if (tid < (int)(sizeof(JssInst) / 16))
        reinterpret_cast<uint4 *>(c.si)[tid] = reinterpret_cast<const uint4 *>(&d)[tid];
    // pools are padded so whole uint4 copies stay in-bounds
    if (what & JSS_STAGE_OPS) {
        {
            const uint4 *src = reinterpret_cast<const uint4 *>(p.ops_pool + d.ops_off);
            uint4 *dst = reinterpret_cast<uint4 *>(c.ops);
            const int n = (d.J * d.M + 7) >> 3;
            for (int k = tid; k < n; k += nt) dst[k] = src[k];
        }
        {
            const uint4 *src = reinterpret_cast<const uint4 *>(p.len_pool + d.len_off);
            uint4 *dst = reinterpret_cast<uint4 *>(c.len);
            const int n = (d.J + 3) >> 2;
            for (int k = tid; k < n; k += nt) dst[k] = src[k];
        }
    }
    if (what & JSS_STAGE_REM) {
        const uint4 *src = reinterpret_cast<const uint4 *>(p.rem_pool + d.rem_off);
        uint4 *dst = reinterpret_cast<uint4 *>(c.rem);
        const int n = (d.J * (d.M + 1) + 7) >> 3;
        for (int k = tid; k < n; k += nt) dst[k] = src[k];
    }
}

// a CTA-uniform work item of instance `inst`: stage its tables (`what`) unless `staged` is that instance already, then
// refresh iv's J / M; returns the instance staged now
JSS_DEV int jss_restage(const JssParams &p, const JssCtaSmem &c, InstView &iv, int inst, int staged, int what) {
    if (inst != staged) {
        __syncthreads();
        jss_stage_instance(p, p.inst[inst], c, what);
        staged = inst;
        __syncthreads();
    }
    jss_iv_shape(iv);
    return staged;
}

template <int KJ, bool BULK = false, bool DIRTY = false>
JSS_DEV void env_emit_all(const JssParams &p, const InstView &iv, const EnvRegs<KJ> &s, int env, int lane,
                          float *scratch, int raw, jss_saddr_t scratch_sa = jss_saddr_t(), void *st_dst = nullptr,
                          jss_saddr_t st_sa = jss_saddr_t(), uint32_t st_bytes = 0u) {
    const JssOut out = jss_out_default(p);
    env_emit_obs<KJ, BULK, DIRTY>(p, out, iv, s, env, lane, scratch, scratch_sa, st_dst, st_sa, st_bytes);
    env_emit_mask<KJ>(p, out, iv, s, env, lane, (s.flags & JSS_FLAG_NOOP_LEGAL) != 0u);
    env_emit_scalars<KJ>(out, iv, s, env, lane, raw);
}

// a step that changed nothing but the sticky error bit: store the new flags word (in the header, the last 4 words of
// the block) and a zero-reward scalar record
template <int KJ>
JSS_DEV void env_store_flags_only(const JssParams &p, const InstView &iv, int32_t *blk, const EnvRegs<KJ> &s, int env,
                                  int lane) {
    if (lane == 0) {
        blk[iv.si->block_words - 4 + JSS_HDR_FLAGS] = (int32_t)s.flags;
        reinterpret_cast<int4 *>(p.scalars)[env] =
            make_int4(0, 0, s.t, (int)((s.flags << 8) | (s.flags & JSS_FLAG_DONE)));
    }
}

// The end of a priority rollout: the whole block and every output if a decision changed the env, else the flags and a
// zero-reward record if they changed.
template <int KJ>
JSS_DEV void env_store_rollout_end(const JssParams &p, const InstView &iv, int32_t *blk, const EnvRegs<KJ> &s, int env,
                                   int lane, float *scratch, bool dirty, int raw, uint32_t flags_in) {
    if (dirty) {
        env_store<KJ>(iv, blk, lane, s);
        env_emit_all<KJ>(p, iv, s, env, lane, scratch, raw);
    } else if (s.flags != flags_in) {
        env_store_flags_only<KJ>(p, iv, blk, s, env, lane);
    }
}

// slot i's first operation not drawn yet: todo, or todo + 1 while the drawn operation todo runs (tufco > 0)
template <int KJ>
JSS_DEV int env_undrawn(const EnvRegs<KJ> &s, int i) { return s.todo[i] + (s.tufco[i] > 0 ? 1 : 0); }

// The gradient of a sampled episode's log-probability with respect to its env's table entries, into `grad` (one row of
// stride ms per job): G[j][k] = sum over the decisions t where job j is legal at operation k of (1[j drawn at t] -
// p_t(j)).  A job is legal only at its current operation, which it leaves only after being drawn there, so each owned
// slot adds up its p_t in a register and puts 1 - acc when drawn (draw), and 0 - acc at its first undrawn operation at
// the end (finish, +0 for a job never legal): one 4-byte access per decision, and the table of gradients is never read
// but by the adds.  Every access to a job's row comes from the lane that owns the job, so program order orders them.
// ADD (the replays of jss_sample_episodes_grad): a put adds w times the value; else it stores the value.
// ENT: the same for the episode's entropy beside it, in a second register per slot: hacc adds up the decisions' q_t(j)
// = p_t(j) (lp_t(j) + H_t) (JssEnt), and G_H = 0 - hacc is put where G is.  ADD adds w G + v G_H (w G first, so that a
// replay with v = 0 adds what the plain replay adds); else G goes to grad and G_H to hgrad, each skipped where NULL.
template <int KJ, bool ADD, bool ENT = false>
struct JssGradAcc {
    float *grad;
    int ms;
    float w;
    float acc[KJ];
    float *hgrad;            // ENT, stored form: the entropy's table
    float v;                 // ENT, ADD: the entropy's weight
    float hacc[KJ];
    JSS_DEV bool on() const { return grad || (ENT && hgrad); }
    JSS_DEV void put(int j, int k, float val, float hval = 0.0f) {
        float *q = grad + (size_t)j * ms + k;
        if (ADD) {
            float t = *q + w * val;
            if (ENT) t += v * hval;
            *q = t;
        } else {
            if (!ENT || grad) *q = val;
            if (ENT && hgrad) hgrad[(size_t)j * ms + k] = hval;
        }
    }
    JSS_DEV void clear() {
#pragma unroll
        for (int i = 0; i < KJ; i++) {
            acc[i] = 0.0f;
            if (ENT) hacc[i] = 0.0f;
        }
    }
    // job `act` (< J) drawn, the owned slots' probabilities pr (ENT: and the decision's gradient terms ent->q)
    JSS_DEV void draw(const EnvRegs<KJ> &s, int lane, int act, const float (&pr)[KJ], const JssEnt<KJ> *ent = nullptr) {
#pragma unroll
        for (int i = 0; i < KJ; i++) {
            acc[i] += pr[i];
            if constexpr (ENT) hacc[i] += ent->q[i];
            if (KJ * lane + i == act) {
                put(act, s.todo[i], 1.0f - acc[i], ENT ? 0.0f - hacc[i] : 0.0f);
                acc[i] = 0.0f;
                if (ENT) hacc[i] = 0.0f;
            }
        }
    }
    JSS_DEV void finish(const EnvRegs<KJ> &s, int lane, int J, int M) {
#pragma unroll
        for (int i = 0; i < KJ; i++) {
            const int j = KJ * lane + i, k0 = env_undrawn<KJ>(s, i);
            if (j < J && k0 < M) put(j, k0, 0.0f - acc[i], ENT ? 0.0f - hacc[i] : 0.0f);
        }
    }
};

// jss_rollout_priority: decisions (env_priority_action) until the episode ends, at most a.n_steps, without reset; a
// done env is left as it is.  Bad priorities set the sticky error bit and end the env's call in its state before that
// decision.  The outputs are written once at the end and equal what the jss_step_greedy calls the loop replaces leave:
// the whole block and every output if a decision changed the env, else the flags and a zero-reward record if they
// changed (the rollout's store covers only the first case, which its rules never leave).
// SAMPLE (jss_rollout_priority_sample): the draws of env_priority_sample_action, decision d with h = jss_hash3(seed,
// global env id, sample_counter + d).  Besides those outputs: log_prob_out[env], the sum of the decisions'
// log-probabilities in decision order (NaN if a decision of this call left the env unchanged with the error bit), and,
// with grad_out, the gradient of that sum with respect to the env's table entries (JssGradAcc).  The operations drawn
// before the call get 0, the first undrawn one at the end -acc and the later ones 0; an env that errs gets 0
// everywhere, so that a caller who masks it out gets no NaN in a backward pass.
// ENT (jss_rollout_priority_sample_entropy): also entropy_out[env], the fp32 sum of the decisions' entropies in
// decision order (NaN where log_prob_out is), and, with entropy_grad_out, its gradient by the same rules (JssGradAcc).
template <int KJ, bool SAMPLE, bool ENT = false>
JSS_DEV void env_priority_rollout(const JssParams &p, const JssLaunch &a, const InstView &iv, EnvRegs<KJ> &s, int32_t *blk,
                                  int env, int lane, float *scratch) {
    const int J = jss_J(iv), M = jss_M(iv);
    JssGradAcc<KJ, false, ENT> g{SAMPLE && a.grad_out ? a.grad_out + (size_t)env * p.jobs_max * p.machines_max : nullptr,
                                 p.machines_max, 1.0f, {}};
    if constexpr (ENT)
        g.hgrad = a.entropy_grad_out ? a.entropy_grad_out + (size_t)env * p.jobs_max * p.machines_max : nullptr;
    const auto zero_ops = [&](int i, int k0, int k1) {   // operations k0 .. k1-1 of owned slot i
        for (int k = k0; k < k1; k++) g.put(KJ * lane + i, k, 0.0f);
    };
    if (g.on()) {
#pragma unroll
        for (int i = 0; i < KJ; i++)
            if (KJ * lane + i < J) zero_ops(i, 0, (s.flags & JSS_FLAG_DONE) ? M : env_undrawn<KJ>(s, i));
    }
    const uint64_t genv = p.env_id_base + (uint64_t)env;
    const uint32_t flags_in = s.flags;
    bool dirty = false;
    int raw = 0;                                         // the raw reward in the scalar record
    bool err = false;
    float lp = 0.0f, hs = 0.0f;
    for (int k = 0; k < a.n_steps && !(s.flags & JSS_FLAG_DONE); k++) {
        float logp = 0.0f, pr[KJ];
        JssEnt<KJ> e;
        int act;
        if (SAMPLE) {
            const uint32_t h = jss_hash_env(jss_hash_key_folded(a.seed_folded, a.sample_counter + (uint64_t)k), genv);
            act = jss_uniform(env_priority_sample_action<KJ, ENT>(a, iv, s, env, lane, h, logp, pr, &e));
        } else {
            act = jss_uniform(env_priority_action<KJ>(a, iv, s, env, lane));
        }
        if (act == JSS_ACTION_SKIP) break;               // nothing legal: no decision changes the env
        const uint32_t flags_before = s.flags;
        int r = 0;
        bool changed = false;
        if (act == JSS_INF) {
            s.flags |= JSS_FLAG_ERROR;
        } else {
            if (g.on() && act < J) g.draw(s, lane, act, pr, &e);   // a job drawn (act == J, the no-op, has no p_t)
            changed = env_step<KJ>(p, iv, s, env, lane, act, r, reinterpret_cast<int *>(scratch));
        }
        s.flags = jss_uniform(s.flags);
        if (changed) {
            lp += logp;
            if (ENT) hs += e.h;
            raw = r; dirty = true; continue;
        }
        // unchanged, with the error bit (bad priorities, or a no-op without a pending event): every later decision
        // would find the same state.  A new bit comes with a zero-reward record (env_store_flags_only); the call's
        // log-probability is NaN.
        err = true;
        if (s.flags != flags_before) raw = 0;
        break;
    }
    if (SAMPLE) {
        if (g.on()) {
            if (!err) g.finish(s, lane, J, M);
#pragma unroll
            for (int i = 0; i < KJ; i++)
                if (KJ * lane + i < J) zero_ops(i, err ? 0 : env_undrawn<KJ>(s, i) + 1, M);
        }
        if (lane == 0) a.log_prob_out[env] = err ? JSS_F32_NAN : lp;
        if (ENT && lane == 0) a.entropy_out[env] = err ? JSS_F32_NAN : hs;
    }
    env_store_rollout_end<KJ>(p, iv, blk, s, env, lane, scratch, dirty, raw, flags_in);
}

// What warp `warp` of `tile` works on, and where that env's state block lives.  The kernels recompute it where they
// store the block instead of carrying it in registers across a step or a rollout.
struct JssTileWarp {
    int env;                 // -1: the tile has fewer envs than warp + 1
    int inst;                // the tile's instance
    uint32_t off16, blk16;   // the env's state block: offset and size in 16-byte units
};
// uni: every env runs the instance `a.uni` (a compile-time constant in the step kernels).  Then env = 8 * tile + warp
// and its block lies at env * block16: no descriptor load.  Otherwise one 16-byte JssTile load (blocks in tile order).
JSS_DEV JssTileWarp jss_tile(const JssParams &p, const JssLaunch &a, bool uni, int tile, int warp) {
    JssTileWarp t;
    if (uni) {
        const int e = tile * JSS_WARPS_PER_CTA + warp;
        t.env = e < p.n_envs ? e : -1;
        t.inst = p.uniform_inst;
        t.blk16 = (uint32_t)a.uni.block_words >> 2;
        t.off16 = (uint32_t)e * t.blk16;
    } else {
        const int4 td = *reinterpret_cast<const int4 *>(p.tiles + tile);
        t.inst = td.y >> 8;
        t.env = warp < (td.y & 255) ? p.order[td.x + warp] : -1;
        t.blk16 = (uint32_t)td.w;
        t.off16 = (uint32_t)td.z + (uint32_t)warp * t.blk16;
    }
    return t;
}

// ---- one-step lookahead over a rule, a priority table or a logit table (jss_lookahead, _priority, _sample) -------
// Work item (tile, sp) of a launch split S ways (a.split): warp `warp` values its env of the tile at the (candidate,
// sample) pairs q = sp, sp + S, ... < (J + 1) K, candidate c = q / K and sample s = q % K (K = 1 but for the sampled
// kind, so that the other two loop over the candidates c = sp, sp + S, ... <= J).  Each pair is simulated in registers
// from the env's state block, which the call never writes: load, step c, then the kind's decisions d = 0, 1, ... until
// done, every step with env_step<KJ, false>.  Lane 0 stores the end time at column q of the env's row of a.values_out,
// or -1 for an illegal candidate, an env done at entry, and a rollout that stops before done (nothing is legal, a step
// leaves the env unchanged with the error bit, a bad table entry, or the bound trips).  The block is reloaded for each
// pair (unchanged and L2-resident) instead of kept as a second register copy of the root state.
// JSS_LOOK_RULE (jss_lookahead): the rule's decisions, RNG counter step_index + d, at most 2 J M + 1 of them.
// JSS_LOOK_TABLE (jss_lookahead_priority): env_priority_action's on the caller's table (a.table), no RNG, at most
//   2 J M + 1.  A bad table at a decision (JSS_INF) stops that candidate's rollout and touches nothing else.
// JSS_LOOK_SAMPLE (jss_lookahead_sample): env_priority_sample_action's draws on the caller's logit table, K =
//   a.n_samples, decision d of sample s at RNG counter sample_counter + s B + d, B = 2 jobs_max machines_max + 1, as
//   env_sample_episodes draws them, and at most B of them.  Every candidate of an env sees the same numbers.
#define JSS_LOOK_RULE 0
#define JSS_LOOK_TABLE 1
#define JSS_LOOK_SAMPLE 2
template <int KJ, int KIND>
JSS_DEV void env_lookahead(const JssParams &p, const JssLaunch &a, const InstView &iv, int env, int tile, int warp,
                           int lane, int sp, float *scratch) {
    constexpr bool SAMPLE = KIND == JSS_LOOK_SAMPLE;
    const int32_t *blk = p.state + (size_t)jss_tile(p, a, p.uniform_inst >= 0, tile, warp).off16 * 4;
    int32_t *out = a.values_out + (int64_t)env * a.out_ld;
    const uint64_t genv = p.env_id_base + (uint64_t)env;
    const int J = jss_J(iv), bound = SAMPLE ? 2 * p.jobs_max * p.machines_max + 1 : 2 * J * jss_M(iv) + 1;
    const int K = SAMPLE ? a.n_samples : 1, pairs = (J + 1) * K;   // below 2^31: jss_lookahead_sample checks it
    int *hz = reinterpret_cast<int *>(scratch);
    for (int q = sp; SAMPLE ? q < pairs : q <= J; q += a.split) {
        const int c = SAMPLE ? q / K : q, smp = SAMPLE ? q % K : 0;
        const uint64_t c0 = a.sample_counter + (uint64_t)smp * (uint64_t)bound;
        EnvRegs<KJ> s;
        env_load<KJ>(iv, blk, lane, s);
        s.flags = jss_uniform(s.flags);
        const uint32_t bits = __shfl_sync(JSS_FULL, s.lb, c < J ? c / KJ : 0);
        const bool legal = !(s.flags & JSS_FLAG_DONE) &&
                           (c < J ? ((bits >> (c % KJ)) & 1u) != 0u : (s.flags & JSS_FLAG_NOOP_LEGAL) != 0u);
        int t = -1;
        if (legal) {
            int r;
            bool ok = env_step<KJ, false>(p, iv, s, env, lane, c, r, hz);
            s.flags = jss_uniform(s.flags);
            for (int d = 0; ok && !(s.flags & JSS_FLAG_DONE) && d < bound; d++) {
                int act;
                if (KIND == JSS_LOOK_TABLE) {
                    act = jss_uniform(env_priority_action<KJ>(a, iv, s, env, lane));
                } else if (SAMPLE) {
                    const uint32_t h = jss_hash_env(jss_hash_key_folded(a.seed_folded, c0 + (uint64_t)d), genv);
                    float logp, pr[KJ];
                    act = jss_uniform(env_priority_sample_action<KJ>(a, iv, s, env, lane, h, logp, pr));
                } else {
                    const uint32_t h = jss_hash3(a.seed, genv, a.step_index + (uint64_t)d);
                    act = jss_uniform(env_select_action<KJ>(iv, s, lane, a.rule, a.coin_mode, h, a.cr_factor));
                }
                ok = act != JSS_ACTION_SKIP && !(KIND != JSS_LOOK_RULE && act == JSS_INF) &&
                     env_step<KJ, false>(p, iv, s, env, lane, act, r, hz);
                s.flags = jss_uniform(s.flags);
            }
            if (s.flags & JSS_FLAG_DONE) t = s.t;
        }
        if (lane == 0) out[q] = t;
    }
}

// ---- K episodes per env drawn from a logit table, the envs untouched (jss_sample_episodes, _grad, _solution) -----
// Sample s of env `env` is jss_rollout_priority_sample's loop run in registers from the env's state block, which the
// call never writes: at most B = 2 jobs_max machines_max + 1 decisions of env_priority_sample_action, decision d at RNG
// counter a.sample_counter + s B + d, each step with env_step<KJ, false>.  It ends done, errs (a bad table, or a
// step that leaves the env unchanged: log-probability NaN) or stops (nothing legal, or the bound).  The block is
// reloaded for each sample, as the lookahead reloads it for each candidate.
// JSS_MODE_SAMPLE_EPISODES: work item (tile, sp) of a launch split S ways (a.split) takes the samples s = sp, sp + S,
//   ... < K and stores each one's makespan (-1 unless done) and log-probability at column s of the env's rows of
//   a.makespan_out and a.log_prob_out; an env done at entry gets -1 and 0 in each of those columns.
// JSS_MODE_SAMPLE_EPISODES_GRAD: work item (tile, c), c < a.split, takes the samples s = c, c + split, ... in
//   increasing s and adds w_s G_s into chunk c of a.grad_out with JssGradAcc<KJ, true>: w_s (1 - acc) at a drawn
//   operation, w_s (0 - acc) at each job's first undrawn one at the end.  Each entry is read and written
//   only by the lane that owns its job, in program order, so a chunk's sums do not depend on the schedule.  A sample
//   that errs adds nothing.  Only a non-finite table entry or an imported legal job without an operation can make a
//   sample err after its first draw (a no-op is drawn only from an imported state, at decision 0, before any add), so
//   an env with either has each sample first run without adds to find out.  Samples with w_s == 0 and envs done at
//   entry are skipped.
// JSS_MODE_SAMPLE_EPISODES_SOLUTION: one work item per tile; env i replays sample a.sample_in[i] (none if < 0) and writes
//   the start time of each operation it starts into a.solution_out.
// JSS_MODE_ORDER_LOG_PROB / _GRAD: the loop of JSS_MODE_SAMPLE_EPISODES / _GRAD with the decisions of env_order_action
//   on order s of the env (a.order_in) in place of the draws; no RNG.
// The _ENT forms of these modes also store each sample's or order's entropy (0 for an env done at entry, NaN where the
// log-probability is NaN) at its column of a.entropy_out; their _GRAD replays add w_s G_s + v_s G_H,s, v_s from
// a.entropy_weights, and skip a sample only where both weights are 0.
JSS_HD constexpr bool jss_mode_samples(int mode) {
    return mode == JSS_MODE_SAMPLE_EPISODES || mode == JSS_MODE_SAMPLE_EPISODES_GRAD ||
           mode == JSS_MODE_SAMPLE_EPISODES_SOLUTION || mode == JSS_MODE_ORDER_LOG_PROB ||
           mode == JSS_MODE_ORDER_LOG_PROB_GRAD || mode == JSS_MODE_SAMPLE_EPISODES_ENT ||
           mode == JSS_MODE_SAMPLE_EPISODES_ENT_GRAD || mode == JSS_MODE_ORDER_LOG_PROB_ENT ||
           mode == JSS_MODE_ORDER_LOG_PROB_ENT_GRAD;
}
template <int KJ, bool ROW = false, bool ENT = false>
JSS_DEV bool env_table_logp(const JssLaunch &a, const EnvRegs<KJ> &s, int env, int lane, float (&lp)[KJ],
                            float *ent = nullptr);
// Env `env`'s next decision under an operation order `ord` (row stride machines_max; jss_order_log_prob): that of
// env_priority_action on the table -ord, the legal job whose current operation has the smallest entry, ties to the
// lowest job.  Writes logp, its log-probability under the logit table a.table by env_table_logp (so that a beam's score
// and the order's log-probability agree bit for bit), and each owned slot's p_i = exp(lp_i) (0 for a job that is not
// legal).  Returns as env_priority_sample_action does: the no-op, logp and p left 0, when no job is legal and it is;
// JSS_INF for a bad table row; JSS_ACTION_SKIP when nothing is legal.
// SWAP (jss_improve_orders): the entries at ord index sw.x and sw.y read as sw.z and sw.w (an index < 0 matches
// nothing), and the decision is returned without reading a table (logp and p stay 0).
// ENT: also the decision's entropy and gradient terms into *ent, as env_priority_sample_action<KJ, true> writes them.
template <int KJ, bool SWAP = false, bool ENT = false>
JSS_DEV int env_order_action(const JssLaunch &a, const InstView &iv, const EnvRegs<KJ> &s, int env, int lane,
                             const int32_t *ord, int mstride, float &logp, float (&pr)[KJ], int4 sw = int4(),
                             JssEnt<KJ> *ent = nullptr) {
    constexpr uint32_t LM = jss_legal_mask<KJ>();
    logp = 0.0f;
#pragma unroll
    for (int i = 0; i < KJ; i++) pr[i] = 0.0f;
    if constexpr (ENT) jss_ent_clear<KJ>(ent);
    if (!__any_sync(JSS_FULL, (s.lb & LM) != 0u))
        return (s.flags & JSS_FLAG_NOOP_LEGAL) ? jss_J(iv) : JSS_ACTION_SKIP;
    int act = JSS_INF;
    env_legal_argmax<KJ>(s, lane, jss_J(iv), false, [&](int i, int j) {
        if constexpr (SWAP) {
            const int q = j * mstride + jss_sel<KJ>(s.todo, i);
            return -(float)(q == sw.x ? sw.z : q == sw.y ? sw.w : ord[q]);
        }
        return -(float)ord[(size_t)j * mstride + jss_sel<KJ>(s.todo, i)];
    }, act);
    if (SWAP) return act;
    float lp[KJ];
    if (!env_table_logp<KJ, false, ENT>(a, s, env, lane, lp, ENT ? &ent->h : nullptr)) return JSS_INF;
    float la = 0.0f;
#pragma unroll
    for (int i = 0; i < KJ; i++) {
        if ((s.lb >> i) & 1u) pr[i] = jss_fast_exp(lp[i]);
        if (KJ * lane + i == act) la = lp[i];
        if constexpr (ENT) ent->q[i] = pr[i] > 0.0f ? pr[i] * (lp[i] + ent->h) : 0.0f;
    }
    logp = __shfl_sync(JSS_FULL, la, act / KJ);
    return act;
}
template <int KJ, int MODE>
JSS_DEV void env_sample_episodes(const JssParams &p, const JssLaunch &a, const InstView &iv, int env, int tile,
                                 int warp, int lane, int sp, float *scratch) {
    constexpr bool ENT = MODE == JSS_MODE_SAMPLE_EPISODES_ENT || MODE == JSS_MODE_SAMPLE_EPISODES_ENT_GRAD ||
                         MODE == JSS_MODE_ORDER_LOG_PROB_ENT || MODE == JSS_MODE_ORDER_LOG_PROB_ENT_GRAD;
    constexpr bool ORD = MODE == JSS_MODE_ORDER_LOG_PROB || MODE == JSS_MODE_ORDER_LOG_PROB_GRAD ||
                         MODE == JSS_MODE_ORDER_LOG_PROB_ENT || MODE == JSS_MODE_ORDER_LOG_PROB_ENT_GRAD;
    constexpr bool GRAD = MODE == JSS_MODE_SAMPLE_EPISODES_GRAD || MODE == JSS_MODE_ORDER_LOG_PROB_GRAD ||
                          MODE == JSS_MODE_SAMPLE_EPISODES_ENT_GRAD || MODE == JSS_MODE_ORDER_LOG_PROB_ENT_GRAD;
    constexpr bool SOL = MODE == JSS_MODE_SAMPLE_EPISODES_SOLUTION;
    const int32_t *blk = p.state + (size_t)jss_tile(p, a, p.uniform_inst >= 0, tile, warp).off16 * 4;
    const uint64_t genv = p.env_id_base + (uint64_t)env;
    const int J = jss_J(iv), M = jss_M(iv), bound = 2 * p.jobs_max * p.machines_max + 1;
    const int64_t row = (int64_t)env * a.out_ld;
    int *hz = reinterpret_cast<int *>(scratch);
    EnvRegs<KJ> s;
    env_load<KJ>(iv, blk, lane, s);
    s.flags = jss_uniform(s.flags);
    int first = sp, end = a.n_samples, stride = a.split;
    if (SOL) {
        first = jss_uniform(a.sample_in[env]);
        end = first + 1; stride = 1;
        if (first < 0) return;
    }
    if (s.flags & JSS_FLAG_DONE) {
        if (!GRAD && !SOL && lane == 0)
            for (int k = first; k < end; k += stride) {
                a.makespan_out[row + k] = -1;
                a.log_prob_out[row + k] = 0.0f;
                if (ENT) a.entropy_out[row + k] = 0.0f;
            }
        return;
    }
    JssGradAcc<KJ, true, ENT> g{GRAD ? a.grad_out + ((size_t)sp * p.n_envs + env) * p.jobs_max * p.machines_max
                                     : nullptr, p.machines_max, 0.0f, {}};
    bool check = false;                                  // GRAD: a sample may err after an add
    if (GRAD) {
        const float *tab = jss_table_row(a.table, env);
        bool clean = true;
#pragma unroll 1
        for (int i = 0; i < KJ; i++) {
            const int j = KJ * lane + i;
            if (j >= J) break;
            clean = clean && !(((s.lb >> i) & 1u) && jss_sel<KJ>(s.op, i) == JSS_OP_NONE);
            for (int k = 0; k < M; k++) {
                const float x = jss_table_at(a.table, tab, j, k);
                clean = clean && x > -JSS_F32_INF && x < JSS_F32_INF;
            }
        }
        check = __any_sync(JSS_FULL, !clean);
    }
    for (int smp = first; smp < end; smp += stride) {
        float w = 0.0f, v = 0.0f;
        if (GRAD) {
            w = __int_as_float(jss_uniform(__float_as_int(a.weights[row + smp])));
            if (ENT) v = __int_as_float(jss_uniform(__float_as_int(a.entropy_weights[row + smp])));
            if (w == 0.0f && v == 0.0f) continue;
        }
        const uint64_t c0 = a.sample_counter + (uint64_t)smp * (uint64_t)bound;
        const int32_t *ord = ORD ? a.order_in + ((size_t)env * a.n_samples + smp) * p.jobs_max * p.machines_max : nullptr;
        // GRAD: pass 0 (only where `check`) finds out whether the sample errs, pass 1 adds
        for (int pass = (GRAD && !check) ? 1 : 0; pass < (GRAD ? 2 : 1); pass++) {
            const bool add = GRAD && pass == 1;
            env_load<KJ>(iv, blk, lane, s);
            s.flags = jss_uniform(s.flags);
            g.w = w;
            g.v = v;
            g.clear();
            bool err = false;
            float lp = 0.0f, hs = 0.0f;
            for (int d = 0; d < bound && !(s.flags & JSS_FLAG_DONE); d++) {
                float logp, pr[KJ];
                JssEnt<KJ> e;
                int act;
                if (ORD) {
                    act = jss_uniform(env_order_action<KJ, false, ENT>(a, iv, s, env, lane, ord, p.machines_max, logp,
                                                                       pr, int4(), &e));
                } else {
                    const uint32_t h = jss_hash_env(jss_hash_key_folded(a.seed_folded, c0 + (uint64_t)d), genv);
                    act = jss_uniform(env_priority_sample_action<KJ, ENT>(a, iv, s, env, lane, h, logp, pr, &e));
                }
                if (act == JSS_ACTION_SKIP) break;       // nothing legal: no decision changes the env
                int r;
                bool changed = false;
                if (act != JSS_INF) {
                    if (add && act < J) g.draw(s, lane, act, pr, &e);   // a job drawn (the no-op has no p_t)
                    changed = env_step<KJ, false, false, SOL>(p, iv, s, env, lane, act, r, hz, a.solution_out);
                }
                s.flags = jss_uniform(s.flags);
                if (!changed) { err = true; break; }
                lp += logp;
                if (ENT) hs += e.h;
            }
            if (!GRAD && !SOL && lane == 0) {
                a.makespan_out[row + smp] = (s.flags & JSS_FLAG_DONE) ? s.t : -1;
                a.log_prob_out[row + smp] = err ? JSS_F32_NAN : lp;
                if (ENT) a.entropy_out[row + smp] = err ? JSS_F32_NAN : hs;
            }
            if (err) break;                              // GRAD: no adds, or none yet (decision 0 of pass 1)
            if (add) g.finish(s, lane, J, M);
        }
    }
}

// ---- beam search over a logit table, the envs untouched (jss_beam_search) -----------------------------------------
// Each owned legal job's log-probability under the table, lp[i] = (x - mx) - log(sum exp(x - mx)) over the legal jobs,
// with the loads, reductions and fast exp / log of env_priority_sample_action in the same order, so that lp of the job
// it draws equals its logp bit for bit.  Kept apart from it: with one softmax shared by the two and one loop shared
// by the rollouts and the sampled-episode replays, those calls ran 1-4 % slower on an H100 (DESIGN.md section 4).
// At least one job must be legal; returns false for a bad row (the bad-table rule of env_priority_sample_action).
// ROW (jss_beam_step): x_j is column j of env `env`'s logit row (a.rows) in place of the table entry of job j's current
// operation; everything else is the same.
// ENT: also the decision's entropy into *ent (jss_softmax_entropy on the same d, exponentials, sum and log).
template <int KJ, bool ROW, bool ENT>
JSS_DEV bool env_table_logp(const JssLaunch &a, const EnvRegs<KJ> &s, int env, int lane, float (&lp)[KJ], float *ent) {
    const float *row = ROW ? a.rows + (int64_t)env * a.rows_ld : jss_table_row(a.table, env);
    bool bad = false;                                    // a legal entry is NaN or +inf
    uint32_t xkey = 0u;                                  // 0: below every candidate's key
    float x[KJ];
#pragma unroll
    for (int i = 0; i < KJ; i++) {
        x[i] = 0.0f;
        if ((s.lb >> i) & 1u) {
            x[i] = ROW ? row[KJ * lane + i] : jss_table_at(a.table, row, KJ * lane + i, s.todo[i]);
            bad = bad || !(x[i] < JSS_F32_INF);
            xkey = max(xkey, jss_f32_key(x[i]));
        }
    }
    const float mx = jss_key_f32(__reduce_max_sync(JSS_FULL, xkey));
    if (__any_sync(JSS_FULL, bad) || mx == -JSS_F32_INF) return false;
    float sum = 0.0f, e[KJ];
#pragma unroll
    for (int i = 0; i < KJ; i++) {
        x[i] -= mx;
        e[i] = 0.0f;
        if ((s.lb >> i) & 1u) {
            e[i] = jss_fast_exp(x[i]);
            sum += e[i];
        }
    }
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) sum += __shfl_xor_sync(JSS_FULL, sum, off);   // the same sum in every lane
    const float ls = jss_fast_log(sum);
    if constexpr (ENT) *ent = jss_softmax_entropy<KJ>(x, e, sum, ls);
#pragma unroll
    for (int i = 0; i < KJ; i++) lp[i] = x[i] - ls;
    return true;
}

// Candidate key of the selection order: score descending (jss_f32_key of score + 0, so -0 and +0 tie), then parent slot
// ascending, then job ascending -- the larger key is the better candidate, and no two candidates of a round share one.
// The low word holds ~(parent << 8 | job), 13 bits, which the u16 backpointer of a round keeps.
JSS_DEV uint64_t jss_beam_key(uint32_t score_key, int parent, int job) {
    return ((uint64_t)score_key << 32) | (uint32_t)~(uint32_t)(parent << 8 | job);
}

// The beam region of the CTA's shared memory for width W and state blocks of `bw` words (jss_block_geom of the batch
// maxima): [blocks: 2][W][bw] int32 | [cand: W][W] u64 | [sel: W] u64 | [score: 2][W] f32 | [cnt: W] i32 | [bad] i32,
// and for the stochastic beam search (swor) then [cscore: W][W] f32 | [key: 2][W] f32, the candidates' scores and the
// slots' keys.  jss_beam_search and jss_sample_without_replacement size it with the same function; jss_beam_step with
// one buffer of blocks (nbuf = 1: the parents; the children go straight to their slots' blocks in global memory).
struct JssBeamSmem {
    int32_t *blocks;
    uint64_t *cand, *sel;
    float *score;
    int32_t *cnt, *bad;
    float *cscore, *key;
};
JSS_HD inline size_t jss_beam_smem(char *base, int W, int bw, JssBeamSmem *b, bool swor = false, int nbuf = 2) {
    const size_t o_cand = (size_t)nbuf * W * bw * 4, o_sel = o_cand + (size_t)8 * W * W, o_score = o_sel + (size_t)8 * W;
    const size_t o_cnt = o_score + (size_t)8 * W, o_bad = o_cnt + (size_t)4 * W, end = (o_bad + 4 + 15) & ~(size_t)15;
    const size_t o_key = end + (size_t)4 * W * W, end_swor = (o_key + (size_t)8 * W + 15) & ~(size_t)15;
    if (b) {
        b->blocks = reinterpret_cast<int32_t *>(base);
        b->cand = reinterpret_cast<uint64_t *>(base + o_cand);
        b->sel = reinterpret_cast<uint64_t *>(base + o_sel);
        b->score = reinterpret_cast<float *>(base + o_score);
        b->cnt = reinterpret_cast<int32_t *>(base + o_cnt);
        b->bad = reinterpret_cast<int32_t *>(base + o_bad);
        b->cscore = reinterpret_cast<float *>(base + end);
        b->key = reinterpret_cast<float *>(base + o_key);
    }
    return swor ? end_swor : end;
}

// log(1 - e^x) for x <= 0 (-inf at 0), through expm1 near 0 and log1p below -log 2 (Maechler's split)
JSS_DEV float jss_log1mexp(float x) {
    return x > -0.693147181f ? logf(-expm1f(x)) : log1pf(-expf(x));
}

// Walks the trace of a search with R rounds back from slot `at` of the last round (-1: none) and writes the round at
// which that beam allocates each operation into `ord` (row stride machines_max), -1 for every operation it does not
// allocate; each job's allocations in reverse are its operations M-1, M-2, ... (a complete beam has allocated every
// operation).  Every lane reads the same trace entries.
template <int KJ>
JSS_DEV void jss_beam_order(const JssParams &p, const uint16_t *trace, int W, int R, int J, int M, int lane, int at,
                            int32_t *ord) {
    int seen[KJ];                                        // allocations of each owned job met so far, walking back
#pragma unroll
    for (int i = 0; i < KJ; i++) {
        seen[i] = 0;
        if (KJ * lane + i < J)
            for (int k = 0; k < M; k++) ord[(size_t)(KJ * lane + i) * p.machines_max + k] = -1;
    }
    if (at < 0) return;
    for (int r = R - 1; r >= 0; r--) {
        const uint32_t pj = jss_uniform((uint32_t)trace[(size_t)r * W + at]);   // every lane reads the same entry
        const int j = (int)(pj & 255u);
        at = (int)(pj >> 8);
#pragma unroll
        for (int i = 0; i < KJ; i++)
            if (KJ * lane + i == j) { ord[(size_t)j * p.machines_max + (M - 1 - seen[i])] = r; seen[i]++; }
    }
}

// The pieces of a beam round that jss_beam_search, jss_sample_without_replacement and jss_beam_step share.
// The forced no-ops of a beam: while no job is legal and the no-op is, take it (env_step<KJ, false>; raw: the last
// one's raw reward).  Returns the number taken, or -1 if one leaves the env unchanged.
template <int KJ>
JSS_DEV int env_forced_noops(const JssParams &p, const InstView &iv, EnvRegs<KJ> &s, int env, int lane, int &raw,
                             int *hz) {
    constexpr uint32_t LM = jss_legal_mask<KJ>();
    int n = 0;
    for (; !__any_sync(JSS_FULL, (s.lb & LM) != 0u) && (s.flags & JSS_FLAG_NOOP_LEGAL); n++) {
        const bool ok = env_step<KJ, false>(p, iv, s, env, lane, jss_J(iv), raw, hz);
        s.flags = jss_uniform(s.flags);
        if (!ok) return -1;
    }
    return n;
}

// The expansion of the beam in slot b (state s, some job legal, score sc; SWOR: its key T = bs.key[kb] and the
// round's noise hash hr): the log-probabilities lp of its legal jobs under env `env`'s table or, ROW, logit row
// (env_table_logp), each candidate's score sc + lp and key (jss_f32_key of score + 0; SWOR: the perturbed values G, Z
// and the key in its place, env_beam_search), and the beam's best min(W, candidates) children in key order, by W argmax
// passes, to bs.cand[b W ..] (SWOR: their scores to bs.cscore).  Returns their number, or -1 for a bad row.
template <int KJ, bool SWOR, bool ROW>
JSS_DEV int jss_beam_expand(const JssLaunch &a, const JssBeamSmem &bs, const EnvRegs<KJ> &s, int env, int lane, int b,
                            int W, float sc, int kb, uint32_t hr) {
    float lp[KJ];
    if (!env_table_logp<KJ, ROW>(a, s, env, lane, lp)) return -1;
    uint32_t key[KJ];                                    // 0: not a candidate, or already taken
    int nc = 0;
#pragma unroll
    for (int i = 0; i < KJ; i++) {
        const float cs = sc + lp[i];
        key[i] = ((s.lb >> i) & 1u) && cs > -JSS_F32_INF ? jss_f32_key(cs + 0.0f) : 0u;
        nc += key[i] != 0u;
    }
    if (SWOR) {                                          // the perturbed values G, Z and the keys in their place
        const float T = bs.key[kb];
        float g[KJ];
        uint32_t zk = 0u;
        int zj = 1 << 20;
#pragma unroll
        for (int i = 0; i < KJ; i++) {
            g[i] = (sc + lp[i]) + jss_gumbel(jss_hash_env(hr, (uint64_t)(b * 256 + KJ * lane + i)));
            const uint32_t k = jss_f32_key(g[i] + 0.0f);
            if (key[i] != 0u && k > zk) { zk = k; zj = KJ * lane + i; }
        }
        const uint32_t zbest = __reduce_max_sync(JSS_FULL, zk);
        zj = (int)__reduce_min_sync(JSS_FULL, (unsigned)(zk == zbest ? zj : 1 << 20));
        const float Z = jss_key_f32(zbest);
#pragma unroll
        for (int i = 0; i < KJ; i++) {
            if (key[i] == 0u) continue;
            float kv = T;
            if (KJ * lane + i != zj) {
                const float v = T - g[i] + jss_log1mexp(g[i] - Z);
                kv = fminf(T, T - fmaxf(v, 0.0f) - log1pf(expf(-fabsf(v))));
            }
            key[i] = jss_f32_key(kv + 0.0f);
        }
    }
    const int taken = min(W, (int)__reduce_add_sync(JSS_FULL, (unsigned)nc));
    for (int q = 0; q < taken; q++) {
        uint32_t lk = 0u;
        int lj = 1 << 20;
#pragma unroll
        for (int i = 0; i < KJ; i++)
            if (key[i] > lk) { lk = key[i]; lj = KJ * lane + i; }
        const uint32_t best = __reduce_max_sync(JSS_FULL, lk);
        const int j = (int)__reduce_min_sync(JSS_FULL, (unsigned)(lk == best ? lj : 1 << 20));
#pragma unroll
        for (int i = 0; i < KJ; i++)
            if (KJ * lane + i == j) key[i] = 0u;
        if (lane == 0) bs.cand[b * W + q] = jss_beam_key(best, b, j);
        if (SWOR) {
            float cj = 0.0f;
#pragma unroll
            for (int i = 0; i < KJ; i++)
                if (KJ * lane + i == j) cj = sc + lp[i];
            cj = __shfl_sync(JSS_FULL, cj, j / KJ);
            if (lane == 0) bs.cscore[b * W + q] = cj;
        }
    }
    return taken;
}

// Selection, by the whole CTA: each kept candidate of the n slots' sorted lists (bs.cnt[b] of them) is ranked against
// the others, and rank < W becomes new slot rank in bs.sel (SWOR: its score goes to buffer cur ^ 1 of bs.score).
// Returns the number of candidates.  The caller synchronises the CTA before and after.
template <bool SWOR>
JSS_DEV int jss_beam_rank(const JssBeamSmem &bs, int n, int W, int cur) {
    int total = 0;
    for (int b = 0; b < n; b++) total += bs.cnt[b];
    for (int e = (int)threadIdx.x; e < n * W; e += (int)blockDim.x) {
        const int b = e / W;
        if (e - b * W >= bs.cnt[b]) continue;
        const uint64_t k = bs.cand[e];
        int rank = 0;
        for (int b2 = 0; b2 < n; b2++) {                 // each list is sorted, best first
            const uint64_t *c2 = bs.cand + b2 * W;
            const int n2 = bs.cnt[b2];
            for (int q = 0; q < n2 && c2[q] > k; q++) rank++;
        }
        if (rank < W) {
            bs.sel[rank] = k;
            if (SWOR) bs.score[(cur ^ 1) * W + rank] = bs.cscore[e];
        }
    }
    return total;
}

// One env searched by the whole CTA (`root`: its state block, never written).  The beams are state blocks in shared
// memory, double-buffered: round r reads buffer r & 1 and writes the other.  Per round (R rounds, the operations not
// started at entry; jss_b200.h):
//   1. warp w expands the beams b = w, w + 8, ...: forced no-ops (env_forced_noops, stored back in place; a beam that
//      then has no legal job has no children), then jss_beam_expand on the table;
//   2. the CTA ranks every candidate against the others' sorted lists; rank < W becomes slot rank;
//   3. warp w loads the parent block of each of its new slots, steps the job with env_step<KJ, false> and stores the
//      result in the other buffer; lane 0 records the backpointer parent << 8 | job in the trace (a.beam_trace).
// At the end warp 0 writes the slot outputs and, with a.order_out, walks the trace back from the best slot
// (jss_beam_order).
// SWOR (jss_sample_without_replacement): the stochastic beam search.  Each slot also carries a key T (the root's is 0).
// In step 1 each candidate j of beam b gets G_j = (score_b + lp_j) + g_j, g_j the Gumbel noise of
// jss_hash_env(jss_hash3(seed, global env, step_index + r), b * 256 + j), and Z = max G; the candidate attaining Z
// (lowest job on ties) gets key T_b, every other one min(T_b, T_b - max(v, 0) - log1p(e^-|v|)), v = T_b - G_j +
// log(1 - e^(G_j - Z)).  The selection ranks the keys in place of the scores; step 2 carries the kept candidates'
// scores over, step 3 their keys.  At the end every warp walks the trace back from its slots b = warp, warp + 8, ...
template <int KJ, bool SWOR>
JSS_DEV void env_beam_search(const JssParams &p, const JssLaunch &a, const InstView &iv, int env, const int32_t *root,
                             int warp, int lane, int *hz, char *bsm) {
    constexpr uint32_t LM = jss_legal_mask<KJ>();
    const int W = a.beam_width, bw = jss_block_geom(p.jobs_max, p.machines_max).words;
    const int J = jss_J(iv), M = jss_M(iv), nw = iv.si->block_words;
    JssBeamSmem bs;
    jss_beam_smem(bsm, W, bw, &bs, SWOR);
    const auto slot = [&](int buf, int b) { return bs.blocks + (size_t)(buf * W + b) * bw; };
    uint16_t *trace = a.beam_trace ? a.beam_trace + (size_t)blockIdx.x * W * p.jobs_max * p.machines_max : nullptr;
    __syncthreads();                                     // the previous env's last reads of the region are done
    for (int k = (int)threadIdx.x; k < nw / 4; k += (int)blockDim.x)
        reinterpret_cast<int4 *>(bs.blocks)[k] = reinterpret_cast<const int4 *>(root)[k];
    if (threadIdx.x == 0) {
        bs.score[0] = 0.0f; bs.bad[0] = 0;
        if (SWOR) bs.key[0] = 0.0f;
    }
    __syncthreads();
    EnvRegs<KJ> s;
    env_load<KJ>(iv, bs.blocks, lane, s);
    s.flags = jss_uniform(s.flags);
    const bool done0 = (s.flags & JSS_FLAG_DONE) != 0u;
    int left = 0;                                        // operations not started: R, summed over the warp
#pragma unroll
    for (int i = 0; i < KJ; i++) left += max(0, M - s.todo[i] - (s.tufco[i] > 0 ? 1 : 0));
    const int R = done0 ? 0 : (int)__reduce_add_sync(JSS_FULL, (unsigned)left);
    int n = 1, cur = 0;                                  // live slots, and the buffer that holds them
    for (int r = 0; r < R && n > 0; r++) {
        const uint32_t hr = SWOR ? jss_hash_env(jss_hash_key_folded(a.seed_folded, a.sample_counter + (uint64_t)r),
                                                p.env_id_base + (uint64_t)env) : 0u;
        for (int b = warp; b < n; b += JSS_WARPS_PER_CTA) {   // 1. expand
            int32_t *blk = slot(cur, b);
            env_load<KJ>(iv, blk, lane, s);
            s.flags = jss_uniform(s.flags);
            const float sc = bs.score[cur * W + b];
            int taken = 0;
            if (sc == sc) {                              // NaN: the step into this slot failed (an imported state)
                int raw;
                const int noops = env_forced_noops<KJ>(p, iv, s, env, lane, raw, hz);
                const bool ok = noops >= 0 && __any_sync(JSS_FULL, (s.lb & LM) != 0u);
                if (ok && noops > 0) env_store<KJ>(iv, blk, lane, s);
                if (ok) {
                    taken = jss_beam_expand<KJ, SWOR, false>(a, bs, s, env, lane, b, W, sc, cur * W + b, hr);
                    if (taken < 0) {
                        taken = 0;
                        if (lane == 0) bs.bad[0] = 1;
                    }
                }
            }
            if (lane == 0) bs.cnt[b] = taken;
        }
        __syncthreads();
        const int total = jss_beam_rank<SWOR>(bs, n, W, cur);   // 2. select
        __syncthreads();
        const int nn = min(W, total), nxt = cur ^ 1;
        for (int b = warp; b < nn; b += JSS_WARPS_PER_CTA) {   // 3. step the kept children
            const uint64_t k = bs.sel[b];
            const uint32_t pj = ~(uint32_t)k;
            const int parent = (int)(pj >> 8), j = (int)(pj & 255u);
            env_load<KJ>(iv, slot(cur, parent), lane, s);
            s.flags = jss_uniform(s.flags);
            int raw;
            const bool ok = env_step<KJ, false>(p, iv, s, env, lane, j, raw, hz);
            env_store<KJ>(iv, slot(nxt, b), lane, s);
            if (lane == 0) {
                if (SWOR) {                              // the score came with the selection
                    bs.key[nxt * W + b] = jss_key_f32((uint32_t)(k >> 32));
                    if (!ok) bs.score[nxt * W + b] = JSS_F32_NAN;
                } else {
                    bs.score[nxt * W + b] = ok ? jss_key_f32((uint32_t)(k >> 32)) : JSS_F32_NAN;
                }
                if (trace) trace[(size_t)r * W + b] = (uint16_t)pj;
            }
        }
        __syncthreads();
        n = nn;
        cur = nxt;
    }
    // slot b holds a complete beam
    const auto complete = [&](int b) {
        return !done0 && b < n && (slot(cur, b)[nw - 4 + JSS_HDR_FLAGS] & JSS_FLAG_DONE) &&
               bs.score[cur * W + b] == bs.score[cur * W + b];
    };
    if (SWOR && a.order_out) {
        for (int b = warp; b < W; b += JSS_WARPS_PER_CTA)
            jss_beam_order<KJ>(p, trace, W, R, J, M, lane, complete(b) ? b : -1,
                               a.order_out + ((size_t)env * W + b) * p.jobs_max * p.machines_max);
    }
    if (warp != 0) return;
    // outputs: lane b reports slot b
    const int b = lane;
    int t = -1;
    float sc = -JSS_F32_INF, ky = -JSS_F32_INF;
    if (!done0 && b < n) {
        const int32_t *hdr = slot(cur, b) + nw - 4;
        const float x = bs.score[cur * W + b];
        if ((hdr[JSS_HDR_FLAGS] & JSS_FLAG_DONE) && x == x) {
            t = hdr[JSS_HDR_T]; sc = x;
            if (SWOR) ky = bs.key[cur * W + b];
        }
    }
    const bool any = __any_sync(JSS_FULL, t >= 0);
    if (done0) sc = ky = 0.0f;
    else if (!any && bs.bad[0]) sc = ky = JSS_F32_NAN;
    if (b < W) {
        a.makespan_out[(int64_t)env * a.out_ld + b] = t;
        (SWOR ? a.log_prob_out : a.score_out)[(int64_t)env * a.out_ld + b] = sc;
        if (SWOR) a.key_out[(int64_t)env * a.out_ld + b] = ky;
    }
    if (SWOR || !a.order_out) return;
    // the best slot: smallest makespan, ties to the lowest slot (t < 2^24)
    const int best = any ? (int)(__reduce_min_sync(JSS_FULL, t >= 0 ? ((uint32_t)t << 5) | (uint32_t)b : ~0u) & 31u) : -1;
    jss_beam_order<KJ>(p, trace, W, R, J, M, lane, best, a.order_out + (size_t)env * p.jobs_max * p.machines_max);
}

// ---- one beam-search round per group of W envs from per-beam logit rows (jss_beam_step) ----------------------------
// The whole CTA works on group g (record `rec`: g, its instance, its W slots' block offsets), slot b = env g W + b.  A
// slot is live iff its score (a.score_io) is finite.
//   0. the scores and the live slots' blocks (the parents, as at entry) go to shared memory.  Without a live, not-done
//      slot the group is untouched: parent b, job -1, bad 0, and nothing else is written;
//   1. warp w expands the slots b = w, w + 8, ...: a live, not-done slot with a legal job by jss_beam_expand on its
//      logit row; a bad row sets bad;
//   2. the CTA ranks the candidates (jss_beam_rank);
//   3. warp w steps new slot b = w, w + 8, ... < nn from its parent's block, takes the forced no-ops
//      (env_forced_noops), and writes the slot's block, its observation, mask and scalar record whole (the
//      raw reward of its last step) and its score, parent and job; slots nn .. W-1 get -inf, -1, -1.
// Every step is env_step<KJ, false>: no statistics, solution, auto-reset or RNG.
// SWOR (jss_stochastic_beam_step): the round of env_beam_search<KJ, true>.  Each slot also carries a key T (a.key_io,
// read with the scores); candidate j of the beam in slot b gets G_j, Z and its key exactly as there, with the noise
// jss_hash_env(h, b * 256 + j), h = jss_hash3(seed, env_id_base / W + g, step_index) (the group's global id); the
// selection ranks the keys, and a kept child's score comes with the selection (bs.score[W ..]), its key from it.
template <int KJ, bool SWOR>
JSS_DEV void env_beam_step(const JssParams &p, const JssLaunch &a, const InstView &iv, const int32_t *rec, int warp,
                           int lane, float *scratch, char *bsm) {
    constexpr uint32_t LM = jss_legal_mask<KJ>();
    const int W = a.beam_width, bw = jss_block_geom(p.jobs_max, p.machines_max).words;
    const int nw = iv.si->block_words;
    const int g = rec[0], e0 = g * W;
    const uint32_t *off = reinterpret_cast<const uint32_t *>(rec + 2);
    int *hz = reinterpret_cast<int *>(scratch);
    JssBeamSmem bs;
    jss_beam_smem(bsm, W, bw, &bs, SWOR, 1);
    const auto live = [](float x) { return x > -JSS_F32_INF && x < JSS_F32_INF; };
    __syncthreads();                                     // the previous group's last reads of the region are done
    for (int b = (int)threadIdx.x; b < W; b += (int)blockDim.x) {
        bs.score[b] = a.score_io[e0 + b];
        if (SWOR) bs.key[b] = a.key_io[e0 + b];
    }
    if (threadIdx.x == 0) bs.bad[0] = 0;
    __syncthreads();
    for (int k = (int)threadIdx.x; k < W * (nw / 4); k += (int)blockDim.x) {   // 0. the live slots' blocks
        const int b = k / (nw / 4), q = k - b * (nw / 4);
        if (live(bs.score[b]))
            reinterpret_cast<int4 *>(bs.blocks + (size_t)b * bw)[q] =
                reinterpret_cast<const int4 *>(p.state + (size_t)off[b] * 4)[q];
    }
    __syncthreads();
    bool moves = false;                                  // CTA-uniform: every thread reads the same words
    for (int b = 0; b < W; b++)
        moves = moves || (live(bs.score[b]) && !(bs.blocks[(size_t)b * bw + nw - 4 + JSS_HDR_FLAGS] & JSS_FLAG_DONE));
    if (!moves) {
        for (int b = (int)threadIdx.x; b < W; b += (int)blockDim.x) { a.parent_out[e0 + b] = b; a.job_out[e0 + b] = -1; }
        if (threadIdx.x == 0) a.bad_out[g] = 0;
        return;
    }
    EnvRegs<KJ> s;
    const uint32_t hr = SWOR ? jss_hash_env(jss_hash_key_folded(a.seed_folded, a.sample_counter),
                                            p.env_id_base / (uint64_t)W + (uint64_t)g) : 0u;
    for (int b = warp; b < W; b += JSS_WARPS_PER_CTA) {   // 1. expand
        const float sc = bs.score[b];
        int taken = 0;
        if (live(sc)) {
            env_load<KJ>(iv, bs.blocks + (size_t)b * bw, lane, s);
            s.flags = jss_uniform(s.flags);
            if (!(s.flags & JSS_FLAG_DONE) && __any_sync(JSS_FULL, (s.lb & LM) != 0u)) {
                taken = jss_beam_expand<KJ, SWOR, true>(a, bs, s, e0 + b, lane, b, W, sc, b, hr);
                if (taken < 0) {
                    taken = 0;
                    if (lane == 0) bs.bad[0] = 1;
                }
            }
        }
        if (lane == 0) bs.cnt[b] = taken;
    }
    __syncthreads();
    const int nn = min(W, jss_beam_rank<SWOR>(bs, W, W, 0));   // 2. select (SWOR: the scores to bs.score[W ..])
    __syncthreads();
    for (int b = warp; b < nn; b += JSS_WARPS_PER_CTA) {   // 3. step the kept children into their slots
        const int env = e0 + b;
        const uint64_t k = bs.sel[b];
        const uint32_t pj = ~(uint32_t)k;
        env_load<KJ>(iv, bs.blocks + (size_t)(pj >> 8) * bw, lane, s);
        s.flags = jss_uniform(s.flags);
        int raw;
        bool ok = env_step<KJ, false>(p, iv, s, env, lane, (int)(pj & 255u), raw, hz);
        s.flags = jss_uniform(s.flags);
        ok = ok && env_forced_noops<KJ>(p, iv, s, env, lane, raw, hz) >= 0;
        env_store<KJ>(iv, p.state + (size_t)off[b] * 4, lane, s);
        env_emit_all<KJ>(p, iv, s, env, lane, scratch, raw);
        if (lane == 0) {
            if (SWOR) {                                  // the score came with the selection
                a.score_io[env] = ok ? bs.score[W + b] : JSS_F32_NAN;
                a.key_io[env] = jss_key_f32((uint32_t)(k >> 32));
            } else {
                a.score_io[env] = ok ? jss_key_f32((uint32_t)(k >> 32)) : JSS_F32_NAN;
            }
            a.parent_out[env] = (int)(pj >> 8);
            a.job_out[env] = (int)(pj & 255u);
        }
    }
    for (int b = nn + (int)threadIdx.x; b < W; b += (int)blockDim.x) {   // empty slots: their blocks left stale
        a.score_io[e0 + b] = -JSS_F32_INF;
        if (SWOR) a.key_io[e0 + b] = -JSS_F32_INF;
        a.parent_out[e0 + b] = -1;
        a.job_out[e0 + b] = -1;
    }
    if (threadIdx.x == 0) a.bad_out[g] = bs.bad[0];
}

// ---- critical-path descent on operation orders, the envs untouched (jss_improve_orders) ---------------------------
// The improvement region of the CTA's shared memory for the batch maxima jmax x mmax (row stride mmax throughout):
// [ord: jmax][mmax] i32 | [start: jmax][mmax] i32 | [pairs: jmax * mmax] u32 | [best: 8] u64 | [ctl: 4] i32.  ord is
// the current canonical order, start its operations' start times, pairs the chain's (u << 16 | v) operation pairs,
// best each warp's best neighbour (makespan << 32 | c) and ctl[0] the current makespan, ctl[1] the number of pairs.
struct JssImproveSmem {
    int32_t *ord, *start;
    uint32_t *pairs;
    uint64_t *best;
    int32_t *ctl;
};
JSS_HD inline size_t jss_improve_smem(char *base, int jmax, int mmax, JssImproveSmem *b) {
    const size_t n = (size_t)jmax * mmax * 4, o_best = (3 * n + 15) & ~(size_t)15;
    const size_t o_ctl = o_best + 8 * JSS_WARPS_PER_CTA;
    if (b) {
        b->ord = reinterpret_cast<int32_t *>(base);
        b->start = reinterpret_cast<int32_t *>(base + n);
        b->pairs = reinterpret_cast<uint32_t *>(base + 2 * n);
        b->best = reinterpret_cast<uint64_t *>(base + o_best);
        b->ctl = reinterpret_cast<int32_t *>(base + o_ctl);
    }
    return o_ctl + 16;
}

// One replay of the env whose state block is `root` under an operation order: env_order_action's decisions on `ord`
// (row stride machines_max) with the entries at indices sw.x / sw.y read as sw.z / sw.w, each step with
// env_step<KJ, false>, at most 2 J M + 1 decisions.  Returns the end time if the episode ends done, else -1 (an env done
// at entry, nothing legal, a step that leaves the env unchanged, the bound).  It stops as soon as t reaches `limit`:
// such an episode cannot end below it.  REC: the round of each allocated operation (job allocations counted from 0)
// goes to rec_ord and its start time to rec_start.  rec_ord may be `ord`: an entry is read only while its operation
// is its job's current one, and written once that operation is allocated.
template <int KJ, bool REC>
JSS_DEV int env_improve_replay(const JssParams &p, const JssLaunch &a, const InstView &iv, const int32_t *root,
                               int lane, const int32_t *ord, int4 sw, int limit, int32_t *rec_ord, int32_t *rec_start,
                               int *hz) {
    const int J = jss_J(iv), ms = p.machines_max, bound = 2 * J * jss_M(iv) + 1;
    EnvRegs<KJ> s;
    env_load<KJ>(iv, root, lane, s);
    s.flags = jss_uniform(s.flags);
    if (s.flags & JSS_FLAG_DONE) return -1;
    int round = 0;
    for (int d = 0; d < bound && !(s.flags & JSS_FLAG_DONE) && s.t < limit; d++) {
        float logp, pr[KJ];
        const int act = jss_uniform(env_order_action<KJ, true>(a, iv, s, 0, lane, ord, ms, logp, pr, sw));
        if (act == JSS_ACTION_SKIP) return -1;
        if (REC && act < J) {
#pragma unroll
            for (int i = 0; i < KJ; i++)
                if (KJ * lane + i == act) rec_ord[act * ms + s.todo[i]] = round;
        }
        int r;
        const bool changed = env_step<KJ, false, false, REC>(p, iv, s, 0, lane, act, r, hz, rec_start);
        s.flags = jss_uniform(s.flags);
        if (!changed) return -1;
        round += act < J ? 1 : 0;
    }
    return (s.flags & JSS_FLAG_DONE) ? s.t : -1;
}

// The chain of the canonical schedule (ord, start; row stride machines_max) that ends at makespan T, walked by one
// warp: from the in-call operation (ord >= 0) that ends at T with the largest round, step to the in-call operation on
// the same machine with the largest round below it if that one ends at the current start (recording the pair), else
// to the job predecessor if it is in call and ends there, else stop.  Writes the pairs in walk order and returns their
// number.  Keys (round + 1) << 13 | index fit 27 bits: rounds and indices are below 256 * 32.
template <int KJ>
JSS_DEV int jss_improve_chain(const JssParams &p, const InstView &iv, const int32_t *ord, const int32_t *start,
                              uint32_t *pairs, int T, int lane) {
    const int J = jss_J(iv), M = jss_M(iv), ms = p.machines_max;
    const auto end = [&](int q) { const int j = q / ms; return start[q] + jss_op_d(iv.ops[j * M + q - j * ms]); };
    const auto key = [&](int q) { return ((uint32_t)(ord[q] + 1) << 13) | (uint32_t)q; };
    __syncwarp();                                        // the replay's lanes wrote ord and start
    uint32_t at = 0u;
    for (int j = lane; j < J; j += 32)
        for (int k = 0; k < M; k++)
            if (ord[j * ms + k] >= 0 && end(j * ms + k) == T) at = max(at, key(j * ms + k));
    at = __reduce_max_sync(JSS_FULL, at);
    int n = 0;
    while (at != 0u) {
        const int q = (int)(at & 8191u), r = (int)(at >> 13) - 1, j = q / ms, k = q - j * ms, s0 = start[q];
        const uint32_t m = jss_op_m(iv.ops[j * M + k]);
        uint32_t pm = 0u;                                // the machine predecessor
        for (int jj = lane; jj < J; jj += 32)
            for (int kk = 0; kk < M; kk++) {
                const int rr = ord[jj * ms + kk];
                if (rr >= 0 && rr < r && jss_op_m(iv.ops[jj * M + kk]) == m) pm = max(pm, key(jj * ms + kk));
            }
        pm = __reduce_max_sync(JSS_FULL, pm);
        at = 0u;
        if (pm != 0u && end((int)(pm & 8191u)) == s0) {
            if (lane == 0) pairs[n] = (pm & 8191u) << 16 | (uint32_t)q;
            n++;
            at = pm;
        } else if (k > 0 && ord[q - 1] >= 0 && end(q - 1) == s0) {
            at = key(q - 1);
        }
    }
    return n;
}

// Order `smp` of env `env` (a.order_in, [N][k][jobs_max][machines_max]) improved by steepest descent on the critical
// path, by the whole CTA (`root`: the env's state block, never written).  Warp 0 replays the input recording its
// canonical order R and start times into shared memory, and walks the chain; then per move warp w replays the
// neighbours c = w, w + 8, ... (pair c's two entries of R swapped at lookup), the CTA takes the smallest makespan
// (lowest c on ties) and, if it is below the current one, warp 0 replays that neighbour recording its canonical order
// in place and walks its chain.  At most a.max_moves moves.  Outputs: the final order (-1 everywhere unless the input
// ends done) to a.order_out, and makespan, the input's makespan and the moves at column smp of the env's rows.
template <int KJ>
JSS_DEV void env_improve_order(const JssParams &p, const JssLaunch &a, const InstView &iv, int env, int smp,
                               const int32_t *root, int warp, int lane, int *hz, char *ism) {
    const int J = jss_J(iv), M = jss_M(iv), ms = p.machines_max;
    JssImproveSmem is;
    jss_improve_smem(ism, p.jobs_max, ms, &is);
    const size_t o_off = ((size_t)env * a.n_samples + smp) * p.jobs_max * ms;
    const int64_t row = (int64_t)env * a.out_ld + smp;
    const int4 none = make_int4(-1, -1, 0, 0);
    __syncthreads();                                     // the previous item's last reads of the region are done
    if (warp == 0) {
        for (int q = lane; q < J * ms; q += 32) is.ord[q] = -1;   // the operations started before the call
        __syncwarp();
        const int t = env_improve_replay<KJ, true>(p, a, iv, root, lane, a.order_in + o_off, none, JSS_INF, is.ord,
                                                   is.start, hz);
        const int n = t >= 0 ? jss_improve_chain<KJ>(p, iv, is.ord, is.start, is.pairs, t, lane) : 0;
        if (lane == 0) { is.ctl[0] = t; is.ctl[1] = n; }
    }
    __syncthreads();
    const int t0 = is.ctl[0];
    int cur = t0, moves = 0;
    while (cur >= 0 && moves < a.max_moves) {
        const int n = is.ctl[1];
        uint64_t best = ~0ull;
        for (int c = warp; c < n; c += JSS_WARPS_PER_CTA) {
            const uint32_t pr = is.pairs[c];
            const int u = (int)(pr >> 16), v = (int)(pr & 0xffffu);
            const int t = env_improve_replay<KJ, false>(p, a, iv, root, lane, is.ord,
                                                        make_int4(u, v, is.ord[v], is.ord[u]), cur, nullptr, nullptr, hz);
            if (t >= 0 && t < cur) best = min(best, (uint64_t)t << 32 | (uint32_t)c);
        }
        if (lane == 0) is.best[warp] = best;
        __syncthreads();
        best = ~0ull;
        for (int w = 0; w < JSS_WARPS_PER_CTA; w++) best = min(best, is.best[w]);
        if (best == ~0ull) break;                        // CTA-uniform: a local optimum
        if (warp == 0) {
            const uint32_t pr = is.pairs[(uint32_t)best];
            const int u = (int)(pr >> 16), v = (int)(pr & 0xffffu);
            const int t = env_improve_replay<KJ, true>(p, a, iv, root, lane, is.ord,
                                                       make_int4(u, v, is.ord[v], is.ord[u]), JSS_INF, is.ord,
                                                       is.start, hz);
            const int n2 = jss_improve_chain<KJ>(p, iv, is.ord, is.start, is.pairs, t, lane);
            if (lane == 0) is.ctl[1] = n2;
        }
        cur = (int)(best >> 32);
        moves++;
        __syncthreads();
    }
    int32_t *out = a.order_out + o_off;
    for (int q = (int)threadIdx.x; q < J * M; q += (int)blockDim.x) {
        const int j = q / M, k = q - j * M;
        out[(size_t)j * ms + k] = t0 >= 0 ? is.ord[j * ms + k] : -1;
    }
    if (threadIdx.x == 0) {
        a.makespan_out[row] = cur;
        a.start_out[row] = t0;
        a.moves_out[row] = moves;
    }
}

template <int KJ, int MODE>
JSS_DEV void jss_process_env(const JssParams &p, const JssLaunch &a, const InstView &iv, int env, int tile, int warp,
                             int lane, float *scratch) {
    EnvRegs<KJ> s;
    // the env's state block, derived at each use: with the pointer carried across the rollout loop, bench.py's cfg2
    // recording rollout took 3.88 instead of 3.83 us per transition (median of 3, H100 SXM, 400 W power limit)
    const auto blk = [&]() { return p.state + (size_t)jss_tile(p, a, p.uniform_inst >= 0, tile, warp).off16 * 4; };
    // MODE is a compile-time kernel variant (the hot step kernel carries no policy /
    // rollout / export code); JSS_MODE_RESET instantiates the rarely used rest
    const int mode = (MODE == JSS_MODE_RESET) ? a.mode : MODE;
    int *hz = reinterpret_cast<int *>(scratch);
    if (mode == JSS_MODE_RESET) {
        if (a.env_mask && a.env_mask[env] == 0) return;
        env_reset_regs<KJ>(iv, s, lane);
        env_clear_solution(p, env, lane);
        env_store<KJ>(iv, blk(), lane, s);
        env_emit_all<KJ>(p, iv, s, env, lane, scratch, 0);
        return;
    }
    if (mode == JSS_MODE_IMPORT) {
        if (a.env_mask && a.env_mask[env] == 0) return;
        env_import<KJ>(p, iv, s, env, lane);
        s.ep_steps = 0; s.ep_return = 0;
        env_store<KJ>(iv, blk(), lane, s);
        env_emit_obs<KJ>(p, jss_out_default(p), iv, s, env, lane, scratch);
        env_emit_mask<KJ>(p, jss_out_default(p), iv, s, env, lane, (s.flags & JSS_FLAG_NOOP_LEGAL) != 0u);
        if (lane == 0) p.scalars[4 * (size_t)env + 3] = (int32_t)((s.flags << 8) | (s.flags & JSS_FLAG_DONE));
        return;
    }
    const uint64_t genv = p.env_id_base + (uint64_t)env;
    if (mode == JSS_MODE_POLICY) env_load_for_policy<KJ>(iv, blk(), lane, s, a.rule);
    else env_load<KJ>(iv, blk(), lane, s);
    s.flags = jss_uniform(s.flags);                      // one word read by every lane (see jss_uniform)
    if (mode == JSS_MODE_EXPORT) { env_export<KJ>(p, iv, s, env, lane); return; }
    if (mode == JSS_MODE_PACK) { env_pack<KJ>(a, iv, s, env, lane, scratch); return; }
    if (mode == JSS_MODE_REFRESH) { env_emit_obs<KJ>(p, jss_out_default(p), iv, s, env, lane, scratch); return; }
    if (MODE == JSS_MODE_PRIORITY || MODE == JSS_MODE_PRIORITY_SAMPLE || MODE == JSS_MODE_PRIORITY_SAMPLE_ENT) {
        constexpr bool ENT = MODE == JSS_MODE_PRIORITY_SAMPLE_ENT;
        env_priority_rollout<KJ, MODE == JSS_MODE_PRIORITY_SAMPLE || ENT, ENT>(p, a, iv, s, blk(), env, lane, scratch);
        return;
    }
    if (mode == JSS_MODE_POLICY) {
        const uint32_t h = jss_hash3(a.seed, genv, a.step_index);
        const int act = env_select_action<KJ>(iv, s, lane, a.rule, a.coin_mode, h, a.cr_factor);
        if (lane == 0) a.actions_out[env] = act;
        return;
    }
    if (mode == JSS_MODE_STEP) {
        const int action = jss_uniform(a.actions[env]);
        int raw = 0;
        const uint32_t flags_in = s.flags;
        const bool changed = env_step<KJ>(p, iv, s, env, lane, action, raw, hz);
        s.flags = jss_uniform(s.flags);
        if (changed) {
            env_store<KJ>(iv, blk(), lane, s);
            env_emit_all<KJ>(p, iv, s, env, lane, scratch, raw);
        } else if (s.flags != flags_in) {
            env_store_flags_only<KJ>(p, iv, blk(), s, env, lane);
        }
        if (a.export_after) env_export<KJ>(p, iv, s, env, lane);   // single-env facade: one launch per transition
        return;
    }
    // JSS_MODE_ROLLOUT: n_steps x (policy -> step) with the state held in registers.
    // Trajectory recording (a.traj_obs != NULL): step k of this env writes its observation / mask / scalar record (and
    // the action that led to it) into slot k * n_envs + env of the caller's [n_steps][N][...] buffers -- the emit helpers
    // index their outputs by env only, so a shifted index and other base pointers are all it takes (ONE loop body).
    const bool record = a.traj_obs != nullptr;
    const JssOut out = record ? JssOut{a.traj_obs, a.traj_mask, a.traj_scalars} : jss_out_default(p);
    bool dirty = false;
    int raw = 0;
    for (int k = 0; k < a.n_steps; k++) {
        const uint32_t h = jss_hash3(a.seed, genv, a.step_index + (uint64_t)k);
        const int act = jss_uniform(env_select_action<KJ>(iv, s, lane, a.rule, a.coin_mode, h, a.cr_factor));
        int r = 0;
        const bool changed = env_step<KJ>(p, iv, s, env, lane, act, r, hz);
        s.flags = jss_uniform(s.flags);
        if (changed) { raw = r; dirty = true; }
        if (record || (changed && a.write_obs)) {
            const int slot = record ? k * p.n_envs + env : env;
            if (record && a.traj_actions && lane == 0) a.traj_actions[slot] = act;
            env_emit_obs<KJ>(p, out, iv, s, slot, lane, scratch);
            env_emit_mask<KJ>(p, out, iv, s, slot, lane, (s.flags & JSS_FLAG_NOOP_LEGAL) != 0u);
            env_emit_scalars<KJ>(out, iv, s, slot, lane, changed ? r : 0);
        }
    }
    if (dirty) {
        env_store<KJ>(iv, blk(), lane, s);
        if (!a.write_obs || record) env_emit_all<KJ>(p, iv, s, env, lane, scratch, raw);
    }
}

// ---- the modes of the generic kernel: one row each (JSS_MODES) ---------------------------------------------------
// What one work item of jss_env_kernel's CTA-strided loop is; launch_all counts the items of a class by the same rule.
#define JSS_ITEM_WARP 0    // a tile, one env per warp (the items are the class's tiles themselves)
#define JSS_ITEM_SPLIT 1   // (tile, s), s < S = a.split: warp w takes env w of the tile and share s of its candidates
                           // or samples; a tile's S items are adjacent and share its instance
#define JSS_ITEM_ENV 2     // one env of the class's tiles per CTA
#define JSS_ITEM_ORDER 3   // one (env, order) per CTA: env slot item / K of the class's tiles, order item % K
                           // (K = a.n_samples; 64-bit items)
#define JSS_ITEM_GROUP 4   // one group record of a.beam_groups per CTA (the items are the class's records themselves)
// The grid of a launch over `items` work items with `slots` resident CTAs.
#define JSS_GRID_ALL 0        // one CTA per item: a policy touches ~50 B per env and is latency-bound, so every tile
                              // gets its own CTA instead of a persistent loop with a dependent load per iteration
#define JSS_GRID_RESIDENT 1   // min(items, slots)
#define JSS_GRID_SPREAD_J 2   // the same, with each tile's candidates spread over S items while the tiles alone leave
                              // slots empty: S = 1 once they fill them, up to the class's J + 1 for a small batch
#define JSS_GRID_SPREAD_K 3   // the same, up to S = K samples per tile
#define JSS_GRID_SPREAD_JK 4  // the same, up to S = (the class's J + 1) K (candidate, sample) pairs per tile, with
                              // S = slots / tiles rounded down, so that every item runs in the first wave
// The host stages what the rule reads: ops / len, + the suffix sums for MWR / LWR / CR, no table for the masked-uniform
// sampler (it reads only J)
#define JSS_STAGE_BY_RULE (-1)
// Shared-memory layout families (jss_api.cu): [instance tables][8 per-warp regions][the CTA's region]
#define JSS_SMEM_ENV 0         // every table; per warp the observation staging, which env_check_no_op's table shares
#define JSS_SMEM_BEAM 1        // no suffix sums; per warp env_check_no_op's table; two buffers of W beams (jss_beam_smem)
#define JSS_SMEM_BEAM_STEP 2   // no suffix sums; per warp the observation staging; one buffer of W beams
#define JSS_SMEM_IMPROVE 3     // no suffix sums; per warp env_check_no_op's table; the improvement region
                               // (jss_improve_smem)
// Whether launch_all first rewrites a real_obs that a recording step left stale: a mode that may read or partly
// rewrite real_obs does; one that reads only the state blocks and writes the caller's buffers does not.
#define JSS_REFRESH_NO 0
#define JSS_REFRESH_YES 1
#define JSS_REFRESH_UNLESS_RECORDING 2   // a step recording into the caller's slot (a.traj_obs) does not
struct JssMode {
    int kernel;                       // the JSS_MODE_* whose jss_env_kernel instantiation runs the mode
    int min_ctas[JSS_LANE_CLASSES];   // resident CTAs per SM that kernel is built for, by lane class (launch bound)
    int item, grid, stage, smem;      // JSS_ITEM_*, JSS_GRID_*, JSS_STAGE_*, JSS_SMEM_*
    bool keys;                        // beam layouts: every slot also carries a Gumbel key
    int refresh;                      // JSS_REFRESH_*
};
// Resident CTAs: one, except in the loops that keep an env on chip for a whole episode or rollout, so that more warps
// per SM hide their latency: there a count per lane class that builds without a stack frame or spills.  The notes give
// the registers by class and where one CTA more spills (ptxas, CUDA 12.9, sm_90a).
constexpr JssMode JSS_MODES[] = {
    // RESET also runs a step that exports (facade), export, import, pack and refresh
    {JSS_MODE_RESET, {1, 1, 1, 1}, JSS_ITEM_WARP, JSS_GRID_RESIDENT, JSS_STAGE_OPS, JSS_SMEM_ENV, false, JSS_REFRESH_YES},
    {JSS_MODE_RESET, {1, 1, 1, 1}, JSS_ITEM_WARP, JSS_GRID_RESIDENT, JSS_STAGE_OPS, JSS_SMEM_ENV, false,
     JSS_REFRESH_UNLESS_RECORDING},                                                                       // STEP
    {JSS_MODE_ROLLOUT, {1, 1, 1, 1}, JSS_ITEM_WARP, JSS_GRID_RESIDENT, JSS_STAGE_ALL, JSS_SMEM_ENV, false,
     JSS_REFRESH_YES},
    {JSS_MODE_POLICY, {1, 1, 1, 1}, JSS_ITEM_WARP, JSS_GRID_ALL, JSS_STAGE_BY_RULE, JSS_SMEM_ENV, false, JSS_REFRESH_NO},
    {JSS_MODE_RESET, {1, 1, 1, 1}, JSS_ITEM_WARP, JSS_GRID_RESIDENT, JSS_STAGE_OPS, JSS_SMEM_ENV, false,
     JSS_REFRESH_NO},                                                                                     // EXPORT
    {JSS_MODE_RESET, {1, 1, 1, 1}, JSS_ITEM_WARP, JSS_GRID_RESIDENT, JSS_STAGE_OPS, JSS_SMEM_ENV, false,
     JSS_REFRESH_YES},                                                                                    // IMPORT
    {JSS_MODE_RESET, {1, 1, 1, 1}, JSS_ITEM_WARP, JSS_GRID_RESIDENT, JSS_STAGE_OPS, JSS_SMEM_ENV, false,
     JSS_REFRESH_YES},                                                                                    // PACK
    {JSS_MODE_RESET, {1, 1, 1, 1}, JSS_ITEM_WARP, JSS_GRID_RESIDENT, JSS_STAGE_OPS, JSS_SMEM_ENV, false,
     JSS_REFRESH_NO},                                                                                     // REFRESH
    // the priority loop carries none of the rules' code, 64 / 80 / 80 / 124 registers: one CTA more spills with 1 and 8
    // jobs per lane, not with 2 or 4; its sampling form at 64 / 80 / 64 / 123: with 1, 4 and 8, not with 2
    {JSS_MODE_PRIORITY, {4, 3, 3, 2}, JSS_ITEM_WARP, JSS_GRID_RESIDENT, JSS_STAGE_OPS, JSS_SMEM_ENV, false,
     JSS_REFRESH_YES},
    {JSS_MODE_PRIORITY_SAMPLE, {4, 3, 4, 2}, JSS_ITEM_WARP, JSS_GRID_RESIDENT, JSS_STAGE_OPS, JSS_SMEM_ENV, false,
     JSS_REFRESH_YES},
    // the lookahead loop: the rules' code, but no output emission, 53 / 64 / 78 / 104 registers, one CTA more spills
    // in every class; over a priority table (the table's argmax in place of the rules) 31 / 48 / 56 / 80 registers, one
    // CTA more spills in the classes with 2, 4 and 8 jobs per lane, and 8 is the SM's limit
    {JSS_MODE_LOOKAHEAD, {4, 4, 3, 2}, JSS_ITEM_SPLIT, JSS_GRID_SPREAD_J, JSS_STAGE_ALL, JSS_SMEM_ENV, false,
     JSS_REFRESH_NO},
    {JSS_MODE_LOOKAHEAD_PRIORITY, {8, 5, 4, 3}, JSS_ITEM_SPLIT, JSS_GRID_SPREAD_J, JSS_STAGE_OPS, JSS_SMEM_ENV, false,
     JSS_REFRESH_NO},
    // the sampled episodes: the draws at 32 / 32 / 39 / 72 registers, their replay with the gradient adds (the caller's
    // split) at 59 / 64 / 64 / 120, the solution replay (S = 1) at 40 / 48 / 40 / 72; one CTA more spills in every
    // class below the SM's limit of 8
    {JSS_MODE_SAMPLE_EPISODES, {8, 8, 6, 3}, JSS_ITEM_SPLIT, JSS_GRID_SPREAD_K, JSS_STAGE_OPS, JSS_SMEM_ENV, false,
     JSS_REFRESH_NO},
    {JSS_MODE_SAMPLE_EPISODES_GRAD, {4, 4, 4, 2}, JSS_ITEM_SPLIT, JSS_GRID_RESIDENT, JSS_STAGE_OPS, JSS_SMEM_ENV,
     false, JSS_REFRESH_NO},
    {JSS_MODE_SAMPLE_EPISODES_SOLUTION, {6, 5, 6, 3}, JSS_ITEM_SPLIT, JSS_GRID_RESIDENT, JSS_STAGE_OPS, JSS_SMEM_ENV,
     false, JSS_REFRESH_NO},
    // the beam search: 62 / 75 / 121 / 173 registers, one CTA more spills in every class; its shared memory (2 W state
    // blocks) bounds the resident CTAs at large W anyway.  The stochastic one: 60 / 78 / 118 / 175 registers, the
    // same.
    {JSS_MODE_BEAM_SEARCH, {4, 3, 2, 1}, JSS_ITEM_ENV, JSS_GRID_RESIDENT, JSS_STAGE_OPS, JSS_SMEM_BEAM, false,
     JSS_REFRESH_NO},
    {JSS_MODE_SWOR, {4, 3, 2, 1}, JSS_ITEM_ENV, JSS_GRID_RESIDENT, JSS_STAGE_OPS, JSS_SMEM_BEAM, true, JSS_REFRESH_NO},
    // the order likelihood at 40 / 62 / 64 / 92 registers, its gradient at 64 / 72 / 64 / 124; one CTA more spills in
    // every class of the likelihood, and in the classes with 1, 2 and 4 jobs per lane of the gradient (not with 8)
    {JSS_MODE_ORDER_LOG_PROB, {6, 4, 4, 2}, JSS_ITEM_SPLIT, JSS_GRID_SPREAD_K, JSS_STAGE_OPS, JSS_SMEM_ENV, false,
     JSS_REFRESH_NO},
    {JSS_MODE_ORDER_LOG_PROB_GRAD, {4, 3, 4, 1}, JSS_ITEM_SPLIT, JSS_GRID_RESIDENT, JSS_STAGE_OPS, JSS_SMEM_ENV, false,
     JSS_REFRESH_NO},
    // the beam round of jss_beam_step (DESIGN.md section 4) at 64 / 78 / 128 / 167 registers, and its stochastic form
    // at 80 / 80 / 128 / 165; one CTA more spills with 1 job per lane in both, not in the other classes
    {JSS_MODE_BEAM_STEP, {4, 3, 2, 1}, JSS_ITEM_GROUP, JSS_GRID_RESIDENT, JSS_STAGE_OPS, JSS_SMEM_BEAM_STEP, false,
     JSS_REFRESH_YES},
    {JSS_MODE_STOCHASTIC_BEAM_STEP, {3, 3, 2, 1}, JSS_ITEM_GROUP, JSS_GRID_RESIDENT, JSS_STAGE_OPS, JSS_SMEM_BEAM_STEP,
     true, JSS_REFRESH_YES},
    // the critical-path descent: 32 / 40 / 60 / 116 registers; 8 is the SM's limit, and one CTA more spills with 2, 4
    // and 8 jobs per lane.  Its shared memory (three [J][M] tables) bounds the resident CTAs at large J M.
    {JSS_MODE_IMPROVE_ORDERS, {8, 6, 4, 2}, JSS_ITEM_ORDER, JSS_GRID_RESIDENT, JSS_STAGE_OPS, JSS_SMEM_IMPROVE, false,
     JSS_REFRESH_NO},
    // the sampled lookahead: the lookahead loop with the draws of the sampled episodes, 25 / 31 / 56 / 91 registers; 8
    // is the SM's limit, and one CTA more spills with 4 and 8 jobs per lane
    {JSS_MODE_LOOKAHEAD_SAMPLE, {8, 8, 4, 2}, JSS_ITEM_SPLIT, JSS_GRID_SPREAD_JK, JSS_STAGE_OPS, JSS_SMEM_ENV, false,
     JSS_REFRESH_NO},
    // the entropy forms, each with its twin's items, grid, tables and layout.  Registers by class at these bounds, no
    // stack: the rollout 80 / 80 / 80 / 119 (one CTA fewer than its twin with 1 and 4 jobs per lane, where the twin's
    // count spills); the draws 48 / 48 / 48 / 76 (5 CTAs, not the twin's 8 / 8 / 6, with 1, 2 and 4: 6 spill); their
    // replay 61 / 64 / 64 / 126, the twin's counts; the order likelihood 48 / 62 / 64 / 94 (5, not 6, with 1 job per
    // lane); its gradient 64 / 72 / 89 / 140 (2, not 4, with 4 jobs per lane: 3 spill)
    {JSS_MODE_PRIORITY_SAMPLE_ENT, {3, 3, 3, 2}, JSS_ITEM_WARP, JSS_GRID_RESIDENT, JSS_STAGE_OPS, JSS_SMEM_ENV, false,
     JSS_REFRESH_YES},
    {JSS_MODE_SAMPLE_EPISODES_ENT, {5, 5, 5, 3}, JSS_ITEM_SPLIT, JSS_GRID_SPREAD_K, JSS_STAGE_OPS, JSS_SMEM_ENV, false,
     JSS_REFRESH_NO},
    {JSS_MODE_SAMPLE_EPISODES_ENT_GRAD, {4, 4, 4, 2}, JSS_ITEM_SPLIT, JSS_GRID_RESIDENT, JSS_STAGE_OPS, JSS_SMEM_ENV,
     false, JSS_REFRESH_NO},
    {JSS_MODE_ORDER_LOG_PROB_ENT, {5, 4, 4, 2}, JSS_ITEM_SPLIT, JSS_GRID_SPREAD_K, JSS_STAGE_OPS, JSS_SMEM_ENV, false,
     JSS_REFRESH_NO},
    {JSS_MODE_ORDER_LOG_PROB_ENT_GRAD, {4, 3, 2, 1}, JSS_ITEM_SPLIT, JSS_GRID_RESIDENT, JSS_STAGE_OPS, JSS_SMEM_ENV,
     false, JSS_REFRESH_NO},
};
static_assert(sizeof(JSS_MODES) / sizeof(JSS_MODES[0]) == JSS_NUM_MODES, "one row per JSS_MODE_*");
// a mode that another mode's kernel runs has that kernel's loop, tables, layout and launch bound
constexpr bool jss_modes_agree() {
    for (const JssMode &m : JSS_MODES) {
        const JssMode &k = JSS_MODES[m.kernel];
        bool same = k.kernel == m.kernel && k.item == m.item && k.stage == m.stage && k.smem == m.smem && k.keys == m.keys;
        for (int c = 0; c < JSS_LANE_CLASSES; c++) same = same && k.min_ctas[c] == m.min_ctas[c];
        if (!same) return false;
    }
    return true;
}
static_assert(jss_modes_agree(), "JSS_MODES: a row disagrees with the row of the kernel that runs it");
JSS_HD constexpr int jss_env_min_ctas(int KJ, int mode) { return JSS_MODES[mode].min_ctas[jss_lane_class(32 * KJ)]; }

// One launch of a mode over the work items of one lane class, CTA-strided: [a.tile_begin, a.tile_end) where the items
// are the tiles or group records themselves, else [0, n) decoded by the mode's item shape.  An item restages the
// instance tables when its instance changes, then runs the mode's body.  An empty warp slot is skipped before staging
// where an item is one env (CTA-uniform), after it where a tile's warps share the item.
template <int KJ, int MODE>
__global__ void __launch_bounds__(JSS_WARPS_PER_CTA * 32, jss_env_min_ctas(KJ, MODE))
jss_env_kernel(const JssParams p, const JssLaunch a, const JssSmemLayout sl) {
    constexpr JssMode M = JSS_MODES[MODE];
    constexpr bool BY_INDEX = M.item == JSS_ITEM_WARP || M.item == JSS_ITEM_GROUP;
    constexpr bool PER_WARP = M.item == JSS_ITEM_WARP || M.item == JSS_ITEM_SPLIT;
    using Item = std::conditional_t<M.item == JSS_ITEM_ORDER, int64_t, int>;
    JSS_SMEM_DECL(jss_smem);
    char *sm = reinterpret_cast<char *>(jss_smem);
    JssCtaSmem c;
    InstView iv;
    jss_cta_carve(sl, sm, c, iv);
    const int warp = jss_warp_index(), lane = threadIdx.x & 31;
    float *scratch = reinterpret_cast<float *>(sm + sl.off_warp0 + warp * sl.warp_stride);
    char *region = sm + sl.off_warp0 + JSS_WARPS_PER_CTA * sl.warp_stride;   // the CTA's beam / improvement region
    const Item K = M.item == JSS_ITEM_ORDER ? (Item)a.n_samples : 1;           // items per env slot
    const Item per_tile = M.item == JSS_ITEM_SPLIT ? (Item)a.split : (Item)JSS_WARPS_PER_CTA * K;
    const Item n_items = (Item)(a.tile_end - a.tile_begin) * per_tile;        // the decoded shapes' items
    const int stage = M.stage == JSS_STAGE_BY_RULE ? a.stage : M.stage;   // a policy's tables depend on its rule
    int staged = -1;
    for (Item item = (BY_INDEX ? a.tile_begin : 0) + (Item)blockIdx.x; item < (BY_INDEX ? (Item)a.tile_end : n_items);
         item += (Item)gridDim.x) {
        if constexpr (M.item == JSS_ITEM_GROUP) {
            const int32_t *rec = a.beam_groups + (size_t)item * (a.beam_width + 2);
            staged = jss_restage(p, c, iv, jss_uniform(rec[1]), staged, M.stage);
            env_beam_step<KJ, M.keys>(p, a, iv, rec, warp, lane, scratch, region);
        } else {
            // SPLIT: tile item / S, share item % S; ENV / ORDER: env slot e = item / K of the class's tiles, order item % K
            const Item e = PER_WARP ? item : item / K;
            const int tile = M.item == JSS_ITEM_WARP ? (int)item
                           : M.item == JSS_ITEM_SPLIT ? a.tile_begin + (int)(item / per_tile)
                                                      : a.tile_begin + (int)(e / JSS_WARPS_PER_CTA);
            const int slot = PER_WARP ? warp : (int)(e % JSS_WARPS_PER_CTA);
            const JssTileWarp t = jss_tile(p, a, p.uniform_inst >= 0, tile, slot);
            const int inst = jss_uniform(t.inst), env = jss_uniform(t.env);
            if (!PER_WARP && env < 0) continue;
            staged = jss_restage(p, c, iv, inst, staged, stage);
            if (env < 0) continue;
            const int32_t *blk = p.state + (size_t)t.off16 * 4;
            const int sub = M.item == JSS_ITEM_SPLIT ? (int)(item % per_tile) : (int)(item - e * K);
            if constexpr (M.item == JSS_ITEM_WARP)
                jss_process_env<KJ, MODE>(p, a, iv, env, tile, warp, lane, scratch);
            else if constexpr (M.item == JSS_ITEM_ENV)
                env_beam_search<KJ, M.keys>(p, a, iv, env, blk, warp, lane, reinterpret_cast<int *>(scratch), region);
            else if constexpr (M.item == JSS_ITEM_ORDER)
                env_improve_order<KJ>(p, a, iv, env, sub, blk, warp, lane, reinterpret_cast<int *>(scratch), region);
            else if constexpr (jss_mode_samples(MODE))
                env_sample_episodes<KJ, MODE>(p, a, iv, env, tile, warp, lane, sub, scratch);
            else
                env_lookahead<KJ, MODE == JSS_MODE_LOOKAHEAD_PRIORITY ? JSS_LOOK_TABLE
                                  : MODE == JSS_MODE_LOOKAHEAD_SAMPLE ? JSS_LOOK_SAMPLE : JSS_LOOK_RULE>(
                    p, a, iv, env, tile, warp, lane, sub, scratch);
        }
    }
}

// ---- programmatic dependent launch (PDL) -------------------------------------------------------
// The step kernels are launched with cudaLaunchAttributeProgrammaticStreamSerialization: the NEXT
// launch's CTAs may become resident (and run their prologue: shared-memory carve-up, mbarrier init,
// staging of the read-only instance tables) while this launch drains; jss_pdl_wait() blocks them until
// every memory operation of the preceding grid is visible, so nothing mutable is touched before it.
#ifndef JSS_EMU
JSS_DEV void jss_pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
JSS_DEV void jss_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
#else
JSS_DEV void jss_pdl_launch_dependents() {}
JSS_DEV void jss_pdl_wait() {}
#endif

// ---- the hot kernels: fused step with TMA prefetch ---------------------------------------------
// Persistent CTAs (grid = SMs x resident CTAs), one warp per env of a tile.  Per warp in shared
// memory: an mbarrier, a state-block buffer that receives the NEXT env's block by cp.async.bulk
// while the current env is simulated, and the staging buffers (new state block, observation rows)
// that leave by bulk store (DIRTY kernels: by the warp's own stores of the changed sectors).
// SAMPLE = 1 / 2 additionally picks every env's NEXT action (masked-uniform sampler / any dispatching
// rule) from the freshly computed state, so a policy-driven loop is one launch per step.
// SAMPLE = 3 takes the env's action from the caller's policy logits BEFORE the step (jss_step_logits): the next env's
// logits row is prefetched like its state block, by 4-byte cp.async into the warp's logits slot.
// SAMPLE = 4 is SAMPLE = 3 with the outputs redirected (jss_step_logits_record): the observation goes to the caller's
// rollout slot (a.traj_obs) instead of real_obs, the mask and the scalar record to the slot and the env's buffers, and
// an env the step left unchanged is emitted into the slot as well.
// SAMPLE = 5 / 6 are SAMPLE = 3 / 4 with the epsilon-greedy decode of the row (jss_step_greedy / _record).
JSS_HD constexpr bool jss_step_takes_row(int sample) { return sample >= 3; }   // the action comes from a row (a.rows)
JSS_HD constexpr bool jss_step_records(int sample) { return sample == 4 || sample == 6; }   // into the caller's slot
struct JssWarpSmem {        // per-warp shared-memory regions of the step kernels
    int32_t *state_in, *state_out;
    float *scratch, *logits;
    jss_saddr_t mbar, state_sa, scratch_sa, state_out_sa, logits_sa;
};

// tiles tile, tile + tile_step, ... < tile_end of ONE lane class through the prefetch pipeline
template <int KJ, int SAMPLE, bool UNI>
JSS_DEV void jss_step_tiles(const JssParams &p, const JssLaunch &a, InstView &iv, const JssCtaSmem &c,
                            const JssWarpSmem &w, int warp, int lane, int tile, int tile_end, int tile_step, int &staged,
                            uint32_t &phase) {
    constexpr bool ROW = jss_step_takes_row(SAMPLE), RECORD = jss_step_records(SAMPLE);
    // a uniform batch stepped by its actions or a rule stores only the changed sectors of a row and of a state block,
    // with the warp's own stores (a row step, whose kernel also prefetches the row, has not been measured with it)
    constexpr bool DIRTY = UNI && !ROW;
    int env_next = -1, act_next = 0;
    // start the bulk load of the state block of this warp's env of tile `next` and fetch its action (a row: start the
    // copy of its logits row, columns 0..J, one 4-byte cp.async per column)
    const auto prefetch = [&](int next) {
        env_next = -1;
        if (next >= tile_end) return;
        const JssTileWarp t = jss_tile(p, a, UNI, next, warp);
        env_next = t.env;
        if (env_next >= 0) {
            if (lane == 0) jss_bulk_load(w.state_sa, p.state + (size_t)t.off16 * 4, t.blk16 * 16u, w.mbar);
            if (ROW) {
                const int J = UNI ? a.uni.J : p.inst[t.inst].J;
                const float *src = a.rows + (size_t)env_next * (size_t)a.rows_ld;
                for (int k = lane; k <= J; k += 32) jss_cp_async4(w.logits_sa + 4u * (uint32_t)k, src + k);
                jss_cp_async_commit();
            } else {
                act_next = a.actions[env_next];
            }
        }
    };
    prefetch(tile);
    for (; tile < tile_end; tile += tile_step) {
        if (!UNI)
            staged = jss_restage(p, c, iv, jss_tile(p, a, UNI, tile, warp).inst, staged, SAMPLE == 2 ? a.stage : JSS_STAGE_OPS);
        const int env = UNI ? env_next : jss_uniform(env_next);
        int action = act_next;
        EnvRegs<KJ> s;
        if (env >= 0) {
            jss_mbar_wait(w.mbar, phase);                // this env's block has landed in shared memory
            phase ^= 1u;
            env_load<KJ>(iv, w.state_in, lane, s);
            __syncwarp();                                // every lane has read the buffer
            if (ROW) {
                jss_cp_async_wait();
                __syncwarp();                            // every lane's columns of the logits row have landed
                int act;
                float logp;
                const uint32_t h = jss_hash_env(a.hash_key, p.env_id_base + (uint64_t)env);
                action = SAMPLE >= 5 ? env_greedy_scores<KJ>(iv, s, lane, w.logits, h, a.explore_t, act, logp)
                                     : env_sample_logits<KJ>(iv, s, lane, w.logits, h, act, logp);
                if (lane == 0) {
                    a.actions_out[env] = act;
                    if (a.log_prob_out) a.log_prob_out[env] = logp;
                }
                __syncwarp();                            // every lane has read the row before the next one is copied in
            }
        }
        prefetch(tile + tile_step);
        if (env < 0) continue;
        int raw = 0;
        // the previous env's observation must have left the staging buffer (also aliased by hz); the dirty-sector
        // stores leave it before they return
        if (!DIRTY) {
            if (lane == 0) jss_bulk_store_wait_read();
            __syncwarp();
        }
        // every lane holds the same flags word (one address, loaded by all lanes): say so -- ptxas already sees that
        // for the action and the time, a shuffle of those is folded away
        if (jss_hint_flags<KJ, UNI>()) s.flags = jss_uniform(s.flags);
        const uint32_t flags_in = s.flags, lb_in = s.lb;
        if (DIRTY) s.dirty = 0u;
        const bool changed =
            env_step<KJ, true, DIRTY>(p, iv, s, env, lane, action, raw, reinterpret_cast<int *>(w.scratch));
        if (jss_hint_flags<KJ, UNI>()) s.flags = jss_uniform(s.flags);   // the no-op test returns from inside lane-dependent code
        if (DIRTY) s.dirty |= ((s.lb ^ lb_in) & jss_legal_mask<KJ>()) << JSS_DIRTY_LEGAL;
        if (SAMPLE == 1 || SAMPLE == 2) {
            const uint32_t h = jss_hash_env(a.hash_key, p.env_id_base + (uint64_t)env);   // == jss_hash3(seed, genv, step_index)
            const int nxt = env_select_action<KJ, SAMPLE == 1>(iv, s, lane, a.rule, a.coin_mode, h, a.cr_factor);
            if (lane == 0) a.actions_out[env] = nxt;
        }
        if (RECORD) {
            // The slot is fresh memory: every env's rows go there, an unchanged env's with the zero-reward record of
            // jss_rollout_traj (env_step leaves raw at 0 then).  One body serves both cases: an unchanged env's block is
            // rewritten as it was loaded plus its new flags (what env_store_flags_only leaves) and its mask row as it was
            // last emitted.  With a branch per case, jss_step_mixed_kernel<4, false> needs a 16-byte stack, not 8.
            const JssOut slot{a.traj_obs, a.traj_mask, a.traj_scalars};
            env_store_to<KJ>(iv, w.state_out, lane, s);
            const JssTileWarp t = jss_tile(p, a, UNI, tile, warp);
            // the new state block and the observation rows leave in one bulk group, as in env_emit_all
            env_emit_obs<KJ, true>(p, slot, iv, s, env, lane, w.scratch, w.scratch_sa, p.state + (size_t)t.off16 * 4,
                                   w.state_out_sa, t.blk16 * 16u);
            const bool noop = (s.flags & JSS_FLAG_NOOP_LEGAL) != 0u;
            env_emit_mask<KJ>(p, jss_out_default(p), iv, s, env, lane, noop);
            if (changed || s.flags != flags_in) env_emit_scalars<KJ>(jss_out_default(p), iv, s, env, lane, raw);
            env_emit_mask<KJ>(p, slot, iv, s, env, lane, noop);
            env_emit_scalars<KJ>(slot, iv, s, env, lane, raw);
        } else if (changed && DIRTY) {
            // new state -> shared staging -> the warp's own stores of the changed sectors of the block and the row
            // (the block last: the emit's __syncwarp covers both staging buffers, and the job registers are dead then)
            env_store_to<KJ>(iv, w.state_out, lane, s);
            env_emit_all<KJ, false, true>(p, iv, s, env, lane, w.scratch, raw);
            env_store_dirty_block<KJ>(iv, s, p.state + (size_t)jss_tile(p, a, UNI, tile, warp).off16 * 4, w.state_out,
                                      lane);
        } else if (changed) {
            // new state -> shared staging -> one bulk store (every word of the block is rewritten)
            env_store_to<KJ>(iv, w.state_out, lane, s);
            const JssTileWarp t = jss_tile(p, a, UNI, tile, warp);
            env_emit_all<KJ, true>(p, iv, s, env, lane, w.scratch, raw, w.scratch_sa,
                                   p.state + (size_t)t.off16 * 4, w.state_out_sa, t.blk16 * 16u);
        } else if (s.flags != flags_in) {
            env_store_flags_only<KJ>(p, iv, p.state + (size_t)jss_tile(p, a, UNI, tile, warp).off16 * 4, s, env, lane);
        }
    }
}

JSS_DEV void jss_step_carve(const JssSmemLayout &sl, char *sm, int warp, JssWarpSmem &w) {
    int woff = sl.off_warp0 + warp * sl.warp_stride;
#ifndef JSS_EMU
    // keep the warp's region offset in ONE register instead of letting the optimiser recompute it from threadIdx
    // (S2R + shift + multiply-add) at every use: -1 % on the uniform ta80 step (94.0 -> 93.2 us)
    asm volatile("" : "+r"(woff));
#endif
    char *wbase = sm + woff;
    w.state_in = reinterpret_cast<int32_t *>(wbase + 16);
    w.scratch = reinterpret_cast<float *>(wbase + sl.off_scratch);
    w.mbar = jss_saddr(sm) + woff;   // shared-space addresses
    w.state_sa = w.mbar + 16;
    w.scratch_sa = w.mbar + sl.off_scratch;
    // state-out staging sits right behind the observation staging (both leave by bulk store)
    w.state_out = reinterpret_cast<int32_t *>(w.scratch + sl.scratch_words);
    w.state_out_sa = w.scratch_sa + sl.scratch_words * 4;
    w.logits = reinterpret_cast<float *>(wbase + sl.off_logits);   // behind state-out (layouts of row steps only)
    w.logits_sa = w.mbar + sl.off_logits;
}

// Uniform batch (every env runs the same instance): static strided tiles, the per-instance scalars are
// read from the kernel parameters (constant-bank operands), no CTA barrier after the first staging.
template <int KJ, int SAMPLE>   // 32 * KJ jobs: the largest instances of KJ's lane class
__global__ void __launch_bounds__(JSS_WARPS_PER_CTA * 32, JSS_MIN_CTAS[jss_lane_class(32 * KJ)])
jss_step_kernel(const JssParams p, const JssLaunch a, const JssSmemLayout sl) {
    JSS_SMEM_DECL(jss_smem);
    char *sm = reinterpret_cast<char *>(jss_smem);
    JssCtaSmem c;
    InstView iv;
    jss_cta_carve(sl, sm, c, iv);
    iv.si = &a.uni; iv.staged = false;
    const int warp = jss_warp_index(), lane = threadIdx.x & 31;
    JssWarpSmem w;
    jss_step_carve(sl, sm, warp, w);
    if (lane == 0) jss_mbar_init(w.mbar);
    jss_pdl_launch_dependents();
    // prologue on read-only data (overlaps the tail of the previous launch under PDL); only a rule reads suffix sums
    jss_stage_instance(p, p.inst[p.uniform_inst], c, SAMPLE == 2 ? a.stage : JSS_STAGE_OPS);
    __syncthreads();
    jss_pdl_wait();
    int staged = p.uniform_inst;
    uint32_t phase = 0;
    // Static strided tiles; the env after the current one is known one iteration ahead, which is what
    // the TMA prefetch needs.
    jss_step_tiles<KJ, SAMPLE, true>(p, a, iv, c, w, warp, lane, a.tile_begin + (int)blockIdx.x, a.tile_end,
                                     (int)gridDim.x, staged, phase);
    if (lane == 0) jss_bulk_store_wait_all();            // shared memory must outlive the bulk reads
}

// Mixed batch: ONE persistent launch covers the three lane classes.  Every CTA gets an equal slice of EVERY class
// (tile counts differ by at most one per class, the extras dithered across CTAs), so the launch is balanced without a
// cost model, and walks them class by class -- three complete loops in sequence, so each lane class keeps the register
// allocation of its stand-alone kernel.  All CTAs start with the 100-job class and move on at about the same time:
// the CTAs that share an SM mostly execute the same 20-35 KB loop body (the three together are 67-86 KB, more than
// the instruction cache holds).  Instance tables are re-staged only when the instance changes.
template <int SAMPLE, bool BIG>   // BIG: the batch contains instances with 129..256 jobs (a fourth, 8-jobs-per-lane body)
__global__ void __launch_bounds__(JSS_WARPS_PER_CTA * 32, JSS_MIN_CTAS[BIG ? 3 : 2])
jss_step_mixed_kernel(const JssParams p, const JssLaunch a, const JssSmemLayout sl) {
    JSS_SMEM_DECL(jss_smem);
    char *sm = reinterpret_cast<char *>(jss_smem);
    JssCtaSmem c;
    InstView iv;
    jss_cta_carve(sl, sm, c, iv);
    const int warp = jss_warp_index(), lane = threadIdx.x & 31;
    JssWarpSmem w;
    jss_step_carve(sl, sm, warp, w);
    if (lane == 0) jss_mbar_init(w.mbar);
    jss_pdl_launch_dependents();
    // one 8-byte load per lane class: with two 16-byte loads <2, false> spills 36 / 44 bytes instead of 32 / 32
    const int2 *range = reinterpret_cast<const int2 *>(p.cta_ranges[blockIdx.x].tiles);
    const int2 r3 = range[3], r2 = range[2], r1 = range[1], r0 = range[0];
    jss_pdl_wait();
    int staged = -1;
    uint32_t phase = 0;
    if (BIG) jss_step_tiles<8, SAMPLE, false>(p, a, iv, c, w, warp, lane, r3.x, r3.y, 1, staged, phase);
    jss_step_tiles<4, SAMPLE, false>(p, a, iv, c, w, warp, lane, r2.x, r2.y, 1, staged, phase);
    jss_step_tiles<2, SAMPLE, false>(p, a, iv, c, w, warp, lane, r1.x, r1.y, 1, staged, phase);
    jss_step_tiles<1, SAMPLE, false>(p, a, iv, c, w, warp, lane, r0.x, r0.y, 1, staged, phase);
    if (lane == 0) jss_bulk_store_wait_all();            // shared memory must outlive the bulk reads
}

// ---- SM-driven copy of small results into mapped pinned host memory -------------------------
// (mask + scalar records, ~8 MB per step at N = 65 536).  Posted PCIe writes from the SMs do not
// queue behind the 183 MB observation transfer that occupies the D2H copy engine.
__global__ void jss_copy16_kernel(uint4 *dst, const uint4 *src, size_t n16) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x * blockDim.x)
        dst[i] = src[i];
}

// ---- per-shard statistics ------------------------------------------------------------------
// one thread per warp slot of the tiles [a.tile_begin, a.tile_end); slots past a tile's count hold no env
__global__ void jss_stats_kernel(const JssParams p, const JssLaunch a, unsigned long long *out) {
    // out[0..7] pre-initialised by the host: sums 0, min = ~0ull
    unsigned long long ep = 0, steps = 0, smk = 0, ndone = 0, nerr = 0;
    long long sret = 0;
    unsigned long long mn = ~0ull, mx = 0;
    for (int slot = a.tile_begin * JSS_WARPS_PER_CTA + blockIdx.x * blockDim.x + threadIdx.x;
         slot < a.tile_end * JSS_WARPS_PER_CTA; slot += gridDim.x * blockDim.x) {
        const JssTileWarp t = jss_tile(p, a, p.uniform_inst >= 0, slot / JSS_WARPS_PER_CTA, slot % JSS_WARPS_PER_CTA);
        const int e = t.env;
        if (e < 0) continue;
        const int64_t *acc = p.acc + (size_t)e * 4;
        const int32_t *hdr = p.state + (size_t)(t.off16 + t.blk16) * 4 - 4;   // the block's last 4 words
        ep += (unsigned long long)p.episode_count[e];
        steps += (unsigned long long)acc[0] + (unsigned long long)(((uint32_t)hdr[JSS_HDR_FLAGS] & JSS_FLAG_DONE) ? 0 : hdr[JSS_HDR_EP_STEPS]);
        smk += (unsigned long long)acc[1];
        sret += acc[2];
        if (p.episode_count[e] > 0) {
            const uint64_t mm = (uint64_t)acc[3];
            mn = min(mn, (unsigned long long)(mm >> 32));
            mx = max(mx, (unsigned long long)(mm & 0xffffffffull));
        }
        ndone += ((uint32_t)hdr[JSS_HDR_FLAGS] & JSS_FLAG_DONE) ? 1 : 0;
        nerr += ((uint32_t)hdr[JSS_HDR_FLAGS] & JSS_FLAG_ERROR) ? 1 : 0;
    }
    atomicAdd(&out[0], ep);
    atomicAdd(&out[1], steps);
    atomicAdd(&out[2], smk);
    atomicMin(&out[3], mn);
    atomicMax(&out[4], mx);
    atomicAdd(&out[5], (unsigned long long)sret);
    atomicAdd(&out[6], ndone);
    atomicAdd(&out[7], nerr);
}
