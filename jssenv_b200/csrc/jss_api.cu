// jss_api.cu -- the C-ABI of include/jss_b200.h on top of the sm_90a kernels in
// jss_device.cuh.  Host side only does: validation, packing of the instance tables,
// grouping envs into per-instance tiles, buffer ownership and kernel launches.
// There is no CPU implementation of the environment in this library.
#ifdef JSS_EMU
#include "cuda_shim.h"  // tests/emu: TEST-ONLY host emulation, never defined for the product build
#else
#include <cuda_runtime.h>
#define JSS_SMEM_DECL(name) extern __shared__ uint4 name[]
#define JSS_LAUNCH(kern, grid, block, smem, stream, ...) kern<<<grid, block, smem, stream>>>(__VA_ARGS__)
// launch with programmatic stream serialization (PDL): the kernel may start its prologue while the preceding
// kernel in the stream drains; it calls griddepcontrol.wait before touching anything mutable
template <typename... KArgs, typename... Args>
static cudaError_t jss_launch_pdl(void (*kern)(KArgs...), int grid, int block, size_t smem, cudaStream_t st, Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3((unsigned)block);
    cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}
#define JSS_LAUNCH_PDL(kern, grid, block, smem, stream, ...) jss_launch_pdl(kern, grid, block, smem, stream, __VA_ARGS__)
#endif
#ifdef JSS_EMU
#define JSS_LAUNCH_PDL(kern, grid, block, smem, stream, ...) (JSS_LAUNCH(kern, grid, block, smem, stream, __VA_ARGS__), cudaSuccess)
#endif

#include <algorithm>
#include <array>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <sched.h>
#include <cctype>
#include <map>
#include <mutex>
#include <utility>
#include <vector>

#include "jss_device.cuh"
#include "jss_host.h"

namespace {

std::string g_create_error;

// the dynamic shared memory each kernel is opted in to, by (device, kernel): the attribute belongs to the kernel on its
// device, so every handle of the process shares it (smem_optin)
std::mutex g_optin_mutex;
std::map<std::pair<int, const void *>, size_t> g_smem_optin;

}  // namespace

struct jss_handle {
    int device = -1;
    int n_envs = 0;
    uint32_t create_flags = 0;
    uint64_t env_id_base = 0;
    int sm_count = 0;
    std::string err;
    int64_t launches = 0;
    bool obs_stale = false;                        // a recording step left real_obs behind the state blocks
    double cr_factor = 1.5;                        // CriticalRatio(due_date_factor), dispatching.py:337

    std::vector<JssInst> insts;
    std::vector<int32_t> len;                      // the jobs_length pool (the packed-observation expansion reads it)
    bool loaded = false, assigned = false;

    // device allocations
    std::vector<void *> allocs;
    void *host_block = nullptr;                    // JSS_CREATE_HOST_MIRROR: pinned + mapped block behind the outputs
    int32_t *mirror_actions = nullptr;
    JssInst *d_inst = nullptr;
    uint16_t *d_ops = nullptr, *d_rem = nullptr;
    int32_t *d_len = nullptr;
    unsigned long long *d_stats = nullptr;
    uint16_t *beam_trace = nullptr;                // jss_beam_search's backpointers (first call with an order)
    size_t beam_trace_bytes = 0;
    struct BeamGroups {                            // jss_beam_step's group records of one width (beam_groups)
        int32_t *dev = nullptr;
        int32_t ranges[JSS_LANE_CLASSES][2] = {};  // [ranges[c][0], ranges[c][1]): the records of lane class c
        std::string err;                           // why the width cannot be used ("": it can)
    };
    std::map<int, BeamGroups> beam_groups;         // by width, built by the first call with it

    JssParams p{};
    JssSmemLayout sl_env{}, sl_step{}, sl_step_rem{};   // shared-memory layouts of the generic / step kernels (step: without / with the suffix-sum table)
    JssSmemLayout sl_step_logits{};                // step kernels drawing the action from policy logits (a logits row per warp)
    int32_t class_tiles[JSS_LANE_CLASSES][2] = {};  // [class_tiles[c][0], class_tiles[c][1]): the tiles of lane class c
    int n_tiles = 0;
    std::map<std::pair<const void *, size_t>, int> ctas_per_sm;   // by kernel and dynamic shared memory (filled lazily)
    std::vector<int32_t> env_inst;
    std::vector<uint32_t> env_off16;               // each env's state block, in 16-byte units (tile order)

    // host-buffer stepping
    int32_t *dev_actions = nullptr;
    float *obs_staging = nullptr;                  // pipelined mode: device copy the D2H engine reads from
    uint8_t *wire[2] = {nullptr, nullptr};         // packed mode: two alternating device rows buffers [N][wire_stride]
    int64_t wire_stride = 0;
    cudaStream_t s_compute = nullptr, s_copy = nullptr;
    cudaEvent_t ev_mask = nullptr, ev_staged = nullptr, ev_wire = nullptr, ev_obs[2] = {nullptr, nullptr};
    int pipe_cur = 0;                              // which ev_obs belongs to the latest begin
    bool pipe_ready = false;
};

namespace {

int fail(jss_t *h, int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (h) h->err = buf; else g_create_error = buf;
    return code;
}

#define JSS_CUDA(h, expr)                                                                           \
    do {                                                                                            \
        cudaError_t e_ = (expr);                                                                    \
        if (e_ != cudaSuccess)                                                                      \
            return fail((h), JSS_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_),  \
                        __FILE__, __LINE__);                                                        \
    } while (0)

template <typename T>
int dev_alloc(jss_t *h, T **out, size_t count, bool zero = true) {
    void *ptr = nullptr;
    const size_t bytes = std::max<size_t>(count * sizeof(T), 16);
    JSS_CUDA(h, cudaMalloc(&ptr, bytes));
    h->allocs.push_back(ptr);
    if (zero) JSS_CUDA(h, cudaMemset(ptr, 0, bytes));
    *out = static_cast<T *>(ptr);
    return JSS_OK;
}

inline int round_up(int x, int m) { return (x + m - 1) / m * m; }
size_t smem_bytes(const JssSmemLayout &sl) { return (size_t)sl.off_warp0 + (size_t)JSS_WARPS_PER_CTA * sl.warp_stride; }

// opts `kern` in to `smem` bytes of dynamic shared memory if that is more than 48 KB and more than it has now.  The
// opt-in is one limit per kernel and device, shared by every handle of the process, so it only ever grows: lowering it
// for a smaller layout would make the next launch with a larger one -- of this handle or of another -- fail.
template <typename Kern>
int smem_optin(jss_t *h, Kern kern, size_t smem) {
    if (smem <= 48 * 1024) return JSS_OK;
    std::lock_guard<std::mutex> lock(g_optin_mutex);
    size_t &optin = g_smem_optin[{h->device, reinterpret_cast<const void *>(kern)}];
    if (smem > optin) {
        JSS_CUDA(h, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        optin = smem;
    }
    return JSS_OK;
}

// resident CTAs per SM of `kern` at `smem` bytes of dynamic shared memory; the first call per kernel and size also
// opts the kernel in to them (smem_optin).  Keyed by size too: the rule-sampling step kernels run with and without the
// suffix-sum table.
template <typename Kern>
int ctas_per_sm(jss_t *h, Kern kern, size_t smem, int &per_sm) {
    const void *key = reinterpret_cast<const void *>(kern);
    int &n = h->ctas_per_sm[{key, smem}];
    if (n == 0) {
        if (int rc = smem_optin(h, kern, smem)) return rc;
        JSS_CUDA(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, JSS_WARPS_PER_CTA * 32, smem));
        if (n < 1) { n = 0; return fail(h, JSS_ERR_CUDA, "kernel does not fit on an SM (smem %zu B)", smem); }
    }
    per_sm = n;
    return JSS_OK;
}

typedef void (*JssKernel)(JssParams, JssLaunch, JssSmemLayout);
// the generic kernel by mode and lane class: the instantiation JSS_MODES[mode].kernel
template <size_t... MODE>
std::array<std::array<JssKernel, JSS_LANE_CLASSES>, sizeof...(MODE)> env_kernel_table(std::index_sequence<MODE...>) {
    return {{{jss_env_kernel<1, JSS_MODES[MODE].kernel>, jss_env_kernel<2, JSS_MODES[MODE].kernel>,
              jss_env_kernel<4, JSS_MODES[MODE].kernel>, jss_env_kernel<8, JSS_MODES[MODE].kernel>}...}};
}
const auto env_kernels = env_kernel_table(std::make_index_sequence<JSS_NUM_MODES>());
template <int SAMPLE>
const JssKernel step_kernels[JSS_LANE_CLASSES] = {jss_step_kernel<1, SAMPLE>, jss_step_kernel<2, SAMPLE>,
                                                  jss_step_kernel<4, SAMPLE>, jss_step_kernel<8, SAMPLE>};
// the rules that read the suffix sums
bool jss_rule_wants_rem(int rule) { return rule == JSS_RULE_MWR || rule == JSS_RULE_LWR || rule == JSS_RULE_CR; }

// the fused step kernel: uniform batches by lane class, mixed batches by whether they hold instances with 129..256 jobs
template <int SAMPLE>
JssKernel step_kernel(const jss_t *h) {
    if (h->p.uniform_inst < 0)
        return h->class_tiles[3][1] > h->class_tiles[3][0] ? jss_step_mixed_kernel<SAMPLE, true>
                                                           : jss_step_mixed_kernel<SAMPLE, false>;
    return step_kernels<SAMPLE>[jss_lane_class(h->insts[h->p.uniform_inst].J)];
}

// one fused step launch (PDL).  A uniform batch runs min(tiles, resident CTAs) persistent CTAs over static strided
// tiles; a mixed batch runs one CTA per JssCtaRange, SMs x JSS_MIN_CTAS[2] of them.  Those are all resident unless the
// batch holds instances with 129..256 jobs: that kernel fits one CTA per SM.
int launch_step(jss_t *h, JssLaunch a, cudaStream_t st) {
    // SAMPLE: 0 none, 1 masked-uniform sampler, 2 dispatching rule, 3 action drawn from policy logits before the step,
    // 4 the same draw with the outputs recorded into the caller's slot, 5 / 6 epsilon-greedy decode of the row (as 3 / 4)
    const int sample = a.rows ? (a.greedy ? 5 : 3) + (a.traj_obs ? 1 : 0)
                     : a.actions_out == nullptr ? 0 : (a.rule == JSS_RULE_RANDOM ? 1 : 2);
    static JssKernel (*const by_sample[])(const jss_t *) = {step_kernel<0>, step_kernel<1>, step_kernel<2>,
                                                            step_kernel<3>, step_kernel<4>, step_kernel<5>,
                                                            step_kernel<6>};
    const JssKernel kern = by_sample[sample](h);
    // only the rules that read the suffix sums stage them; the other launches leave their room to the L1
    a.stage = sample == 2 && jss_rule_wants_rem(a.rule) ? JSS_STAGE_ALL : JSS_STAGE_OPS;
    const JssSmemLayout &sl = jss_step_takes_row(sample) ? h->sl_step_logits
                            : a.stage & JSS_STAGE_REM ? h->sl_step_rem : h->sl_step;
    const size_t smem = smem_bytes(sl);
    int per_sm = 0, rc = ctas_per_sm(h, kern, smem, per_sm);
    if (rc) return rc;
    int grid = h->p.n_cta_ranges;
    if (h->p.uniform_inst >= 0) {
        a.tile_begin = 0;
        a.tile_end = (h->n_envs + JSS_WARPS_PER_CTA - 1) / JSS_WARPS_PER_CTA;
        grid = std::min(a.tile_end, h->sm_count * per_sm);
    }
    JSS_CUDA(h, JSS_LAUNCH_PDL(kern, grid, JSS_WARPS_PER_CTA * 32, smem, st, h->p, a, sl));
    JSS_CUDA(h, cudaGetLastError());
    h->launches += 1;
    return JSS_OK;
}

// ranges: the records of each lane class if not its tiles (jss_beam_step's group records)
int launch_all(jss_t *h, JssLaunch a, cudaStream_t st, const int32_t (*ranges)[2] = nullptr);

// the shared-memory layout of a launch of a.mode (JSS_SMEM_*), and in `smem` its size: the CTA's region behind the
// per-warp regions depends on the width or the batch maxima
JssSmemLayout mode_layout(const jss_t *h, const JssLaunch &a, size_t &smem) {
    const JssMode &m = JSS_MODES[a.mode];
    const int bw = jss_block_geom(h->p.jobs_max, h->p.machines_max).words;
    JssSmemLayout sl = h->sl_env;
    if (m.smem != JSS_SMEM_ENV) sl.off_warp0 = sl.off_rem;                      // no suffix sums
    if (m.smem == JSS_SMEM_BEAM || m.smem == JSS_SMEM_IMPROVE) sl.warp_stride = 32 * 4;   // env_check_no_op's table
    smem = smem_bytes(sl);
    if (m.smem == JSS_SMEM_BEAM) smem += jss_beam_smem(nullptr, a.beam_width, bw, nullptr, m.keys);
    if (m.smem == JSS_SMEM_BEAM_STEP) smem += jss_beam_smem(nullptr, a.beam_width, bw, nullptr, m.keys, 1);
    if (m.smem == JSS_SMEM_IMPROVE) smem += jss_improve_smem(nullptr, h->p.jobs_max, h->p.machines_max, nullptr);
    return sl;
}

// the grid of lane class c's launch of a.mode over the tiles (or records) [a.tile_begin, a.tile_end) at `smem` bytes
// (JSS_GRID_*); a launch that spreads its tiles' candidates or samples also gets its split S in a.split
int mode_grid(jss_t *h, JssLaunch &a, int c, size_t smem, int &grid) {
    const JssMode &m = JSS_MODES[a.mode];
    const int n = a.tile_end - a.tile_begin;
    int per_sm = 0;
    if (int rc = ctas_per_sm(h, env_kernels[a.mode][c], smem, per_sm)) return rc;
    const int slots = h->sm_count * per_sm;
    if (m.grid == JSS_GRID_SPREAD_J || m.grid == JSS_GRID_SPREAD_K) {
        const int most = m.grid == JSS_GRID_SPREAD_J ? std::min(h->p.jobs_max, 32 << c) + 1 : a.n_samples;
        a.split = n >= slots ? 1 : std::min(most, (slots + n - 1) / n);
    }
    if (m.grid == JSS_GRID_SPREAD_JK) {   // rounded down: a tile's many pairs make every item long, and a CTA that
                                          // took a second one would double the launch
        const int64_t most = (int64_t)(std::min(h->p.jobs_max, 32 << c) + 1) * a.n_samples;
        a.split = n >= slots ? 1 : (int)std::min<int64_t>(most, slots / n);
    }
    const int64_t items = m.item == JSS_ITEM_SPLIT ? (int64_t)n * a.split
                        : m.item == JSS_ITEM_ENV ? (int64_t)n * JSS_WARPS_PER_CTA
                        : m.item == JSS_ITEM_ORDER ? (int64_t)n * JSS_WARPS_PER_CTA * a.n_samples : n;
    grid = (int)(m.grid == JSS_GRID_ALL ? items : std::min<int64_t>(items, slots));
    return JSS_OK;
}

// rewrite real_obs from the state blocks if a recording step left it stale (jss_refresh_obs)
int refresh_obs(jss_t *h, cudaStream_t st) {
    if (!h->obs_stale) return JSS_OK;
    JssLaunch a{};
    a.mode = JSS_MODE_REFRESH;
    if (int rc = launch_all(h, a, st)) return rc;
    h->obs_stale = false;
    return JSS_OK;
}

// a plain step: the fused step kernel; every other mode: the generic kernel, one launch per lane class present
int launch_all(jss_t *h, JssLaunch a, cudaStream_t st, const int32_t (*ranges)[2]) {
    const JssMode &m = JSS_MODES[a.mode];
    if (m.refresh == JSS_REFRESH_YES || (m.refresh == JSS_REFRESH_UNLESS_RECORDING && !a.traj_obs))
        if (int rc = refresh_obs(h, st)) return rc;
    if (h->p.uniform_inst >= 0) a.uni = h->insts[h->p.uniform_inst];
    if (a.mode == JSS_MODE_STEP && !a.export_after) return launch_step(h, a, st);   // one launch, whatever the mix of lane classes
    a.stage = m.stage != JSS_STAGE_BY_RULE ? m.stage
            : a.rule == JSS_RULE_RANDOM ? 0 : jss_rule_wants_rem(a.rule) ? JSS_STAGE_ALL : JSS_STAGE_OPS;
    size_t smem = 0;
    const JssSmemLayout sl = mode_layout(h, a, smem);
    if (!ranges) ranges = h->class_tiles;
    for (int c = 0; c < JSS_LANE_CLASSES; c++) {
        a.tile_begin = ranges[c][0];
        a.tile_end = ranges[c][1];
        if (a.tile_end <= a.tile_begin) continue;
        int grid = 0;
        if (int rc = mode_grid(h, a, c, smem, grid)) return rc;
        JSS_LAUNCH(env_kernels[a.mode][c], grid, JSS_WARPS_PER_CTA * 32, smem, st, h->p, a, sl);
        JSS_CUDA(h, cudaGetLastError());
        h->launches += 1;
    }
    return JSS_OK;
}

// the action choice of jss_policy / jss_step_sample / jss_rollout / jss_rollout_traj
bool valid_rule_coin(int rule, int coin_mode) {
    return rule >= 0 && rule < JSS_NUM_RULES && (coin_mode == JSS_COIN_DEVICE || coin_mode == JSS_COIN_NEVER);
}

bool bad_ptr(const void *ptr) { return !ptr || ((uintptr_t)ptr & 3u); }

// a caller's (N, J, M) table into t: non-NULL, 4-byte aligned, strides >= 0
int table_arg(jss_t *h, const char *who, const float *ptr, int64_t ld_env, int64_t ld_job, int64_t ld_op, JssTable &t) {
    if (bad_ptr(ptr) || ld_env < 0 || ld_job < 0 || ld_op < 0)
        return fail(h, JSS_ERR_INVALID, "%s: bad table (%p must be non-NULL and 4-byte aligned, strides %lld / %lld / "
                    "%lld >= 0)", who, (const void *)ptr, (long long)ld_env, (long long)ld_job, (long long)ld_op);
    t = JssTable{ptr, ld_env, ld_job, ld_op};
    return JSS_OK;
}

int check_ready(jss_t *h) {
    if (!h) return JSS_ERR_INVALID;
    if (!h->assigned) return fail(h, JSS_ERR_STATE, "jss_load_instances + jss_assign must be called first");
    JSS_CUDA(h, cudaSetDevice(h->device));
    return JSS_OK;
}

// check_ready for an entry point that works on `stream`: it also orders the stream after the latest
// jss_host_step_begin (its step, result copies and observation transfer), which runs on the handle's own streams and
// reads and writes the same state, outputs and action buffer.  The pipeline's own launches on s_compute are ordered
// already.  Nothing to do before the first begin.
int check_ready(jss_t *h, void *stream) {
    if (int rc = check_ready(h)) return rc;
    const cudaStream_t st = (cudaStream_t)stream;
    if (h->pipe_ready && st != h->s_compute) JSS_CUDA(h, cudaStreamWaitEvent(st, h->ev_obs[h->pipe_cur], 0));
    return JSS_OK;
}

// group envs by (KJ class, instance) -> tiles of <= JSS_WARPS_PER_CTA envs of one instance, the largest lane class
// first (the order in which the mixed-batch step kernel walks its slices); sets the class tile ranges of `h`
int plan_tiles(jss_t *h, const int32_t *env_to_inst, std::vector<int32_t> &order, std::vector<JssTile> &tiles,
               size_t &state_words) {
    const int N = h->n_envs;
    order.resize(N);
    for (int e = 0; e < N; e++) order[e] = e;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) {
        const int ka = env_to_inst[a], kb = env_to_inst[b];
        const int ca = jss_lane_class(h->insts[ka].J), cb = jss_lane_class(h->insts[kb].J);
        if (ca != cb) return ca > cb;
        return ka < kb;
    });
    for (auto &r : h->class_tiles) r[0] = r[1] = 0;
    int pos = 0;
    int cur_class = -1;
    uint64_t off16 = 0;                                  // running state offset in 16-byte units
    while (pos < N) {
        const int k = env_to_inst[order[pos]];
        const int c = jss_lane_class(h->insts[k].J);
        const uint32_t block16 = (uint32_t)h->insts[k].block_words / 4;
        int end = pos;
        while (end < N && env_to_inst[order[end]] == k) end++;
        if (c != cur_class) h->class_tiles[c][0] = (int)tiles.size();   // a class's tiles are contiguous
        cur_class = c;
        for (int f = pos; f < end; f += JSS_WARPS_PER_CTA) {
            JssTile t;
            const int cnt = std::min(JSS_WARPS_PER_CTA, end - f);
            t.first = f;
            t.inst_count = (k << 8) | cnt;
            t.state_off16 = (uint32_t)off16;
            t.block16 = block16;
            off16 += (uint64_t)cnt * block16;
            tiles.push_back(t);
        }
        h->class_tiles[c][1] = (int)tiles.size();
        pos = end;
    }
    h->n_tiles = (int)tiles.size();
    if (off16 >= (1ull << 32)) return fail(h, JSS_ERR_UNSUPPORTED, "state exceeds 64 GiB");
    state_words = (size_t)off16 * 4;
    return JSS_OK;
}

// mixed-batch step kernel: every persistent CTA gets an equal slice of EVERY lane class (tile counts differ by at
// most one per class; the extras are dithered with a different phase per class so that no CTA collects them all)
std::vector<JssCtaRange> plan_cta_ranges(const jss_t *h) {
    const int n_cta = std::max(1, std::min(h->n_tiles, h->sm_count * JSS_MIN_CTAS[2]));
    std::vector<JssCtaRange> ranges((size_t)n_cta);
    for (int c = 0; c < JSS_LANE_CLASSES; c++) {
        const int tb = h->class_tiles[c][0], n = h->class_tiles[c][1] - tb;
        const int shift = (c * n_cta) / JSS_LANE_CLASSES;   // CTA that starts this class's Bresenham sequence
        int given = 0;
        for (int k = 0; k < n_cta; k++) {
            const int b = (k + shift) % n_cta;
            const int upto = (int)(((int64_t)(k + 1) * n) / n_cta);
            ranges[b].tiles[c][0] = tb + given; ranges[b].tiles[c][1] = tb + upto;
            given = upto;
        }
    }
    return ranges;
}

// shared-memory layouts: [JssInst][ops u16][len i32][rem u16][per-warp regions], 16-byte aligned regions; ops_max and
// rem_max are the largest ops / suffix-sum tables of the batch's instances
void plan_smem_layouts(jss_t *h, int jmax, int mmax, int ops_max, int rem_max) {
    const JssBlockGeom g = jss_block_geom(jmax, mmax);   // the geometry grows with J and M: batch maxima
    JssSmemLayout sl{};
    sl.off_len = (int32_t)sizeof(JssInst) + round_up(ops_max, 8) * 2;
    sl.off_rem = sl.off_len + round_up(jmax, 4) * 4;
    sl.off_warp0 = sl.off_rem + round_up(rem_max, 8) * 2;
    // observation staging (7 floats per job slot); env_check_no_op (general instances) also keeps its 32-int
    // per-warp machine-horizon table here, so never less than 32 words (tiny instances: 7 * Jcap < 32)
    sl.scratch_words = std::max(7 * g.Jcap, 32);
    h->sl_env = sl;
    h->sl_env.warp_stride = sl.scratch_words * 4;
    h->sl_env.off_scratch = 0;
    h->sl_step_rem = sl;
    h->sl_step_rem.off_scratch = 16 + g.words * 4;                                     // [mbarrier][state-in]
    h->sl_step_rem.warp_stride = h->sl_step_rem.off_scratch + sl.scratch_words * 4 + g.words * 4;   // [scratch][state-out]
    h->sl_step = h->sl_step_rem;                      // launches that stage no suffix sums leave their room to the L1
    h->sl_step.off_warp0 = h->sl_step.off_rem;
    h->sl_step_logits = h->sl_step;                   // + [logits row: jobs_max + 1 floats]
    h->sl_step_logits.off_logits = h->sl_step.warp_stride;
    h->sl_step_logits.warp_stride += round_up(4 * (jmax + 1), 16);
}

// the per-transition outputs, one device allocation each; with JSS_CREATE_HOST_MIRROR all of them (and an action slot)
// in one pinned, device-mapped host block instead (unified addressing: the device pointer equals the host pointer),
// meant for small batches -- the kernels write over PCIe
int alloc_outputs(jss_t *h) {
    JssParams &p = h->p;
    const size_t N = (size_t)p.n_envs, NJ = N * p.jobs_max, NM = N * p.machines_max;
    struct Output { char **slot; size_t bytes; bool mirror_only = false; };
    const Output outputs[] = {
        {(char **)&p.mask, N * p.mask_stride}, {(char **)&p.obs, NJ * 7 * 4}, {(char **)&p.scalars, N * 16},
        {(char **)&p.x_todo, NJ * 4}, {(char **)&p.x_tufco, NJ * 4}, {(char **)&p.x_idle_last, NJ * 4},
        {(char **)&p.x_total_idle, NJ * 4}, {(char **)&p.x_col4, NJ * 4}, {(char **)&p.x_tuam, NM * 4},
        {(char **)&p.x_legal, NJ}, {(char **)&p.x_blocked, NJ}, {(char **)&h->mirror_actions, N * 4, true}};
    if (!(h->create_flags & JSS_CREATE_HOST_MIRROR)) {
        for (const Output &o : outputs)
            if (int rc = o.mirror_only ? JSS_OK : dev_alloc(h, o.slot, o.bytes)) return rc;
        return JSS_OK;
    }
    auto padded = [](size_t bytes) { return (bytes + 255) / 256 * 256; };
    size_t total = 0;
    for (const Output &o : outputs) total += padded(o.bytes);
    JSS_CUDA(h, cudaHostAlloc(&h->host_block, total, cudaHostAllocMapped | cudaHostAllocPortable));
    memset(h->host_block, 0, total);
    void *dev = nullptr;
    JSS_CUDA(h, cudaHostGetDevicePointer(&dev, h->host_block, 0));
    if (dev != h->host_block) return fail(h, JSS_ERR_CUDA, "host mirror needs unified addressing");
    char *b = static_cast<char *>(h->host_block);
    for (const Output &o : outputs) { *o.slot = b; b += padded(o.bytes); }
    return JSS_OK;
}

}  // namespace

extern "C" {

int jss_abi_version(void) { return JSS_ABI_VERSION; }

const char *jss_last_error(const jss_t *h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int64_t jss_launch_count(const jss_t *h) { return h ? h->launches : 0; }

int jss_set_cr_due_date_factor(jss_t *h, double factor) {
    if (!h || !(factor == factor)) return fail(h, JSS_ERR_INVALID, "jss_set_cr_due_date_factor: bad arguments");
    h->cr_factor = factor;
    return JSS_OK;
}

int jss_create(jss_t **out, int device, int n_envs, uint32_t flags, uint64_t env_id_base) {
    if (!out || n_envs <= 0) return fail(nullptr, JSS_ERR_INVALID, "jss_create: bad arguments");
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(nullptr, JSS_ERR_NO_DEVICE,
                    "no CUDA device (%s); this library has no CPU fallback", cudaGetErrorString(e));
    if (device < 0 || device >= ndev)
        return fail(nullptr, JSS_ERR_NO_DEVICE, "device %d out of range (have %d)", device, ndev);
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess)
        return fail(nullptr, JSS_ERR_NO_DEVICE, "cudaGetDeviceProperties failed");
    if (prop.major != 9 || prop.minor != 0)   // sm_90a code runs on compute capability 9.0 only
        return fail(nullptr, JSS_ERR_NO_DEVICE, "device %d is sm_%d%d; this build targets sm_90a (H100)", device,
                    prop.major, prop.minor);
    jss_t *h = new jss_handle();
    h->device = device;
    h->n_envs = n_envs;
    h->create_flags = flags;
    h->env_id_base = env_id_base;
    h->sm_count = prop.multiProcessorCount;
    if (cudaSetDevice(device) != cudaSuccess) {
        delete h;
        return fail(nullptr, JSS_ERR_CUDA, "cudaSetDevice(%d) failed", device);
    }
    *out = h;
    return JSS_OK;
}

void jss_destroy(jss_t *h) {
    if (!h) return;
    cudaSetDevice(h->device);
    if (h->pipe_ready) {
        cudaStreamSynchronize(h->s_compute); cudaStreamSynchronize(h->s_copy);
        cudaEventDestroy(h->ev_mask); cudaEventDestroy(h->ev_staged); cudaEventDestroy(h->ev_wire); cudaEventDestroy(h->ev_obs[0]); cudaEventDestroy(h->ev_obs[1]);
        cudaStreamDestroy(h->s_compute); cudaStreamDestroy(h->s_copy);
    }
    for (void *ptr : h->allocs) cudaFree(ptr);
    if (h->beam_trace) cudaFree(h->beam_trace);
    if (h->host_block) cudaFreeHost(h->host_block);
    delete h;
}

int jss_load_instances(jss_t *h, int n_inst, const int32_t *jobs, const int32_t *machines, const int64_t *offsets,
                       const int32_t *machine, const int32_t *duration) {
    if (!h || n_inst <= 0 || !jobs || !machines || !offsets || !machine || !duration)
        return fail(h, JSS_ERR_INVALID, "jss_load_instances: bad arguments");
    if (h->loaded) return fail(h, JSS_ERR_STATE, "instances already loaded");
    if (n_inst >= (1 << 23)) return fail(h, JSS_ERR_UNSUPPORTED, "too many instances");
    JSS_CUDA(h, cudaSetDevice(h->device));
    std::vector<uint16_t> ops, rem;
    std::vector<int32_t> len;
    h->insts.resize(n_inst);
    for (int k = 0; k < n_inst; k++) {
        const int J = jobs[k], M = machines[k];
        if (J <= 0 || M <= 1)  // asserts at jss_env.py:93-94
            return fail(h, JSS_ERR_INVALID, "instance %d: need jobs > 0 and machines > 1 (got %dx%d)", k, J, M);
        if (J > JSS_MAX_JOBS || M > JSS_MAX_MACHINES)
            return fail(h, JSS_ERR_UNSUPPORTED, "instance %d: %dx%d exceeds the %dx%d kernel limit", k, J, M,
                        JSS_MAX_JOBS, JSS_MAX_MACHINES);
        const int32_t *mm = machine + offsets[k], *dd = duration + offsets[k];
        int64_t max_time_op = 0, max_time_jobs = 0, sum_op = 0;
        JssInst d{};
        d.J = J; d.M = M;
        d.ops_off = (int32_t)ops.size();
        d.len_off = (int32_t)len.size();
        d.rem_off = (int32_t)rem.size();
        ops.resize(ops.size() + round_up(J * M, 8), 0);
        len.resize(len.size() + round_up(J, 4), 0);
        rem.resize(rem.size() + round_up(J * (M + 1), 8), 0);
        for (int j = 0; j < J; j++) {
            int64_t total = 0;
            for (int i = 0; i < M; i++) {
                const int m = mm[j * M + i], t = dd[j * M + i];
                if (m < 0 || m >= M) return fail(h, JSS_ERR_INVALID, "instance %d: machine %d out of range", k, m);
                // Zero-length ops are rejected: the reference itself cannot finish such an episode -- an allocated op of
                // duration 0 never satisfies `was_left_time > 0` (jss_env.py:529), so the job never advances to its
                // next op and is re-legalised on the same machine at the same instant (jss_env.py:616-634).
                if (t < 1 || t > JSS_MAX_DURATION)
                    return fail(h, JSS_ERR_UNSUPPORTED, "instance %d: duration %d outside [1, %d]", k, t,
                                JSS_MAX_DURATION);
                ops[d.ops_off + j * M + i] = (uint16_t)((m << JSS_OP_SHIFT) | t);
                total += t;
                max_time_op = std::max<int64_t>(max_time_op, t);        // jss_env.py:86
            }
            len[d.len_off + j] = (int32_t)total;                        // jss_env.py:87
            sum_op += total;                                            // jss_env.py:88
            max_time_jobs = std::max(max_time_jobs, total);             // jss_env.py:89
            int64_t suffix = 0;
            rem[d.rem_off + j * (M + 1) + M] = 0;
            for (int i = M - 1; i >= 0; i--) {
                suffix += dd[j * M + i];
                rem[d.rem_off + j * (M + 1) + i] = (uint16_t)suffix;    // <= 32 * 2047 < 65536
            }
        }
        d.max_time_op = (int32_t)max_time_op;
        d.max_time_jobs = (int32_t)max_time_jobs;
        d.sum_op = (int32_t)sum_op;
        d.f_mto = (float)d.max_time_op; d.f_mtj = (float)d.max_time_jobs; d.f_sop = (float)d.sum_op; d.f_M = (float)d.M;
        d.r_mto = 1.0f / (float)d.max_time_op;
        d.r_mtj = 1.0f / (float)d.max_time_jobs;
        d.r_sop = 1.0f / (float)d.sum_op;
        d.r_M = 1.0f / (float)d.M;
        const JssBlockGeom g = jss_block_geom(J, M);
        d.Jcap = g.Jcap; d.Mcap = g.Mcap; d.block_words = g.words; d.tail = g.tail;
        h->insts[k] = d;
    }
    int rc;
    if ((rc = dev_alloc(h, &h->d_inst, (size_t)n_inst))) return rc;
    if ((rc = dev_alloc(h, &h->d_ops, ops.size()))) return rc;
    if ((rc = dev_alloc(h, &h->d_len, len.size()))) return rc;
    if ((rc = dev_alloc(h, &h->d_rem, rem.size()))) return rc;
    JSS_CUDA(h, cudaMemcpy(h->d_inst, h->insts.data(), sizeof(JssInst) * n_inst, cudaMemcpyHostToDevice));
    JSS_CUDA(h, cudaMemcpy(h->d_ops, ops.data(), ops.size() * 2, cudaMemcpyHostToDevice));
    JSS_CUDA(h, cudaMemcpy(h->d_len, len.data(), len.size() * 4, cudaMemcpyHostToDevice));
    JSS_CUDA(h, cudaMemcpy(h->d_rem, rem.data(), rem.size() * 2, cudaMemcpyHostToDevice));
    h->len = std::move(len);
    h->loaded = true;
    return JSS_OK;
}

int jss_instance_scalars(jss_t *h, int inst, int64_t out[3]) {
    if (!h || !out || !h->loaded || inst < 0 || inst >= (int)h->insts.size())
        return fail(h, JSS_ERR_INVALID, "jss_instance_scalars: bad arguments");
    out[0] = h->insts[inst].max_time_op;
    out[1] = h->insts[inst].max_time_jobs;
    out[2] = h->insts[inst].sum_op;
    return JSS_OK;
}

int jss_assign(jss_t *h, const int32_t *env_to_inst) {
    if (!h || !env_to_inst) return fail(h, JSS_ERR_INVALID, "jss_assign: bad arguments");
    if (!h->loaded) return fail(h, JSS_ERR_STATE, "jss_load_instances must be called first");
    if (h->assigned) return fail(h, JSS_ERR_STATE, "envs already assigned");
    JSS_CUDA(h, cudaSetDevice(h->device));
    const int N = h->n_envs, n_inst = (int)h->insts.size();
    int jmax = 0, mmax = 0, ops_max = 0, rem_max = 0;
    h->env_inst.assign(env_to_inst, env_to_inst + N);
    std::vector<char> used(n_inst, 0);
    for (int e = 0; e < N; e++) {
        const int k = env_to_inst[e];
        if (k < 0 || k >= n_inst) return fail(h, JSS_ERR_INVALID, "env %d: instance %d out of range", e, k);
        used[k] = 1;
    }
    for (int k = 0; k < n_inst; k++) {
        if (!used[k]) continue;
        jmax = std::max(jmax, h->insts[k].J);
        mmax = std::max(mmax, h->insts[k].M);
        ops_max = std::max(ops_max, h->insts[k].J * h->insts[k].M);
        rem_max = std::max(rem_max, h->insts[k].J * (h->insts[k].M + 1));
    }
    int rc;
    std::vector<int32_t> order;
    std::vector<JssTile> tiles;
    size_t state_words = 0;
    if ((rc = plan_tiles(h, env_to_inst, order, tiles, state_words))) return rc;
    const std::vector<JssCtaRange> ranges = plan_cta_ranges(h);
    h->env_off16.assign(N, 0);
    for (const JssTile &t : tiles)
        for (int w = 0; w < (t.inst_count & 255); w++) h->env_off16[order[t.first + w]] = t.state_off16 + w * t.block16;

    JssParams &p = h->p;
    p.n_envs = N;
    p.jobs_max = jmax;
    p.machines_max = mmax;
    p.mask_stride = round_up(jmax + 1, jss_lane_slots(1 << jss_lane_class(jmax)));   // whole mask stores per lane
    p.create_flags = (int32_t)h->create_flags;
    p.env_id_base = h->env_id_base;
    {
        bool uniform = true;
        for (int e = 0; e < N; e++) uniform = uniform && env_to_inst[e] == env_to_inst[0];
        p.uniform_inst = uniform ? env_to_inst[0] : -1;   // then `order` is the identity (stable sort)
    }
    p.inst = h->d_inst; p.ops_pool = h->d_ops; p.len_pool = h->d_len; p.rem_pool = h->d_rem;
    plan_smem_layouts(h, jmax, mmax, ops_max, rem_max);

    int32_t *d_order = nullptr;
    JssTile *d_tiles = nullptr;
    JssCtaRange *d_ranges = nullptr;
    if ((rc = dev_alloc(h, &d_order, (size_t)N))) return rc;
    if ((rc = dev_alloc(h, &d_tiles, tiles.size()))) return rc;
    if ((rc = dev_alloc(h, &d_ranges, ranges.size()))) return rc;
    JSS_CUDA(h, cudaMemcpy(d_order, order.data(), (size_t)N * 4, cudaMemcpyHostToDevice));
    JSS_CUDA(h, cudaMemcpy(d_tiles, tiles.data(), tiles.size() * sizeof(JssTile), cudaMemcpyHostToDevice));
    JSS_CUDA(h, cudaMemcpy(d_ranges, ranges.data(), ranges.size() * sizeof(JssCtaRange), cudaMemcpyHostToDevice));
    p.order = d_order;
    p.tiles = d_tiles;
    p.cta_ranges = d_ranges;
    p.n_cta_ranges = (int32_t)ranges.size();
    const size_t NJ = (size_t)N * jmax;
    if ((rc = dev_alloc(h, &p.state, state_words))) return rc;
    if ((rc = alloc_outputs(h))) return rc;
    if (h->create_flags & JSS_CREATE_RECORD_SOLUTION) {
        if ((rc = dev_alloc(h, &p.solution, NJ * mmax, false))) return rc;
        JSS_CUDA(h, cudaMemset(p.solution, 0xff, NJ * mmax * 4));  // -1
    } else {
        p.solution = nullptr;
    }
    if ((rc = dev_alloc(h, &p.episode_count, (size_t)N))) return rc;
    if ((rc = dev_alloc(h, &p.last_makespan, (size_t)N))) return rc;
    if ((rc = dev_alloc(h, &p.last_return, (size_t)N))) return rc;
    if ((rc = dev_alloc(h, &p.acc, (size_t)N * 4))) return rc;
    if ((rc = dev_alloc(h, &h->d_stats, (size_t)JSS_STATS_LEN))) return rc;
    if ((rc = dev_alloc(h, &h->dev_actions, (size_t)N))) return rc;
    h->assigned = true;
    // a fresh batch starts reset, like a freshly constructed + reset reference env
    if ((rc = jss_reset(h, nullptr, nullptr))) return rc;
    // the memsets above and this reset run on the legacy default stream, which a caller's non-blocking stream does not
    // wait for: return only once they have completed, so the batch may be stepped at once on any stream
    JSS_CUDA(h, cudaStreamSynchronize(nullptr));
    return JSS_OK;
}

int jss_get_buffers(jss_t *h, jss_buffers *out) {
    if (!h || !out) return JSS_ERR_INVALID;
    if (!h->assigned) return fail(h, JSS_ERR_STATE, "jss_assign must be called first");
    const JssParams &p = h->p;
    memset(out, 0, sizeof *out);
    out->n_envs = p.n_envs; out->jobs_max = p.jobs_max; out->machines_max = p.machines_max;
    out->mask_stride = p.mask_stride;
    out->action_mask = p.mask; out->real_obs = p.obs; out->solution = p.solution;
    out->host_mirror = h->host_block ? 1 : 0;
    out->mirror_actions = h->mirror_actions;
    out->scalar_stride = 16;   // reward / reward_raw / time / flags_done are fields of one 16-byte record per env
    out->reward = reinterpret_cast<float *>(p.scalars); out->reward_raw = p.scalars + 1;
    out->time = p.scalars + 2; out->flags_done = reinterpret_cast<uint32_t *>(p.scalars + 3);
    out->done = reinterpret_cast<uint8_t *>(p.scalars + 3);
    out->episode_count = p.episode_count; out->last_makespan = p.last_makespan; out->last_return = p.last_return;
    out->x_todo = p.x_todo; out->x_tufco = p.x_tufco; out->x_idle_last = p.x_idle_last;
    out->x_total_idle = p.x_total_idle; out->x_col4 = p.x_col4; out->x_tuam = p.x_tuam;
    out->x_legal = p.x_legal; out->x_blocked = p.x_blocked;
    return JSS_OK;
}

int jss_reset(jss_t *h, const uint8_t *env_mask_dev, void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    JssLaunch a{};
    a.mode = JSS_MODE_RESET;
    a.env_mask = env_mask_dev;
    return launch_all(h, a, (cudaStream_t)stream);
}

int jss_step(jss_t *h, const int32_t *actions_dev, void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    if (!actions_dev) return fail(h, JSS_ERR_INVALID, "jss_step: actions_dev is NULL");
    JssLaunch a{};
    a.mode = JSS_MODE_STEP;
    a.actions = actions_dev;
    return launch_all(h, a, (cudaStream_t)stream);
}

int jss_step_export(jss_t *h, const int32_t *actions_dev, void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    if (!actions_dev) return fail(h, JSS_ERR_INVALID, "jss_step_export: actions_dev is NULL");
    JssLaunch a{};
    a.mode = JSS_MODE_STEP;
    a.actions = actions_dev;
    a.export_after = 1;
    return launch_all(h, a, (cudaStream_t)stream);
}

int jss_step_sample(jss_t *h, const int32_t *actions_dev, int rule, int coin_mode, uint64_t seed,
                    uint64_t step_index, int32_t *next_actions_dev, void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    if (!actions_dev || bad_ptr(next_actions_dev) || !valid_rule_coin(rule, coin_mode))
        return fail(h, JSS_ERR_INVALID, "jss_step_sample: bad arguments (rule %d, coin %d)", rule, coin_mode);
    JssLaunch a{};
    a.mode = JSS_MODE_STEP;
    a.actions = actions_dev;
    a.actions_out = next_actions_dev;
    a.rule = rule; a.coin_mode = coin_mode; a.cr_factor = h->cr_factor;
    a.hash_key = jss_hash_key(seed, step_index);
    return launch_all(h, a, (cudaStream_t)stream);
}

namespace {
// the checks and the launch arguments jss_step_logits and jss_step_logits_record share
int logits_launch(jss_t *h, const char *what, const float *logits_dev, int64_t ld, uint64_t seed, uint64_t step_index,
                  int32_t *actions_out_dev, float *log_prob_out_dev, JssLaunch &a) {
    if (!logits_dev || bad_ptr(actions_out_dev) || ld < (int64_t)h->p.jobs_max + 1)
        return fail(h, JSS_ERR_INVALID, "%s: bad arguments (logits %p, actions_out %p, ld %lld < jobs_max + 1 = %d)", what,
                    (const void *)logits_dev, (void *)actions_out_dev, (long long)ld, h->p.jobs_max + 1);
    a = JssLaunch{};
    a.mode = JSS_MODE_STEP;
    a.rows = logits_dev;
    a.rows_ld = ld;
    a.actions_out = actions_out_dev;
    a.log_prob_out = log_prob_out_dev;
    a.hash_key = jss_hash_key(seed, step_index);
    return JSS_OK;
}

// jss_step_greedy / _record: the checks and launch arguments of logits_launch, plus epsilon as the threshold
// T = floor(epsilon 2^32) (exact in double, 0 .. 2^32) of the exploration coin
int greedy_launch(jss_t *h, const char *what, const float *scores_dev, int64_t ld, double epsilon, uint64_t seed,
                  uint64_t step_index, int32_t *actions_out_dev, float *log_prob_out_dev, JssLaunch &a) {
    if (!(epsilon >= 0.0 && epsilon <= 1.0))
        return fail(h, JSS_ERR_INVALID, "%s: epsilon %g is not in [0, 1]", what, epsilon);
    if (int rc = logits_launch(h, what, scores_dev, ld, seed, step_index, actions_out_dev, log_prob_out_dev, a)) return rc;
    a.greedy = 1;
    a.explore_t = (uint64_t)std::floor(epsilon * 4294967296.0);
    return JSS_OK;
}

// the recording step: the caller's slot pointers into `a`, then the launch, which leaves real_obs stale
int launch_record(jss_t *h, const char *what, float *obs_out_dev, uint8_t *mask_out_dev, int32_t *scalars_out_dev,
                  JssLaunch &a, cudaStream_t st) {
    // the kernels store observation rows by bulk copy and scalar records as 16-byte vectors
    const auto aligned = [](const void *ptr) { return ptr && ((uintptr_t)ptr & 15u) == 0; };
    if (!aligned(obs_out_dev) || !aligned(mask_out_dev) || !aligned(scalars_out_dev))
        return fail(h, JSS_ERR_INVALID, "%s: obs_out %p, mask_out %p and scalars_out %p must be 16-byte aligned device "
                    "pointers", what, (void *)obs_out_dev, (void *)mask_out_dev, (void *)scalars_out_dev);
    a.traj_obs = obs_out_dev; a.traj_mask = mask_out_dev; a.traj_scalars = scalars_out_dev;
    if (int rc = launch_all(h, a, st)) return rc;
    h->obs_stale = true;
    return JSS_OK;
}
}  // namespace

int jss_step_logits(jss_t *h, const float *logits_dev, int64_t ld, uint64_t seed, uint64_t step_index,
                    int32_t *actions_out_dev, float *log_prob_out_dev, void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    JssLaunch a;
    if ((rc = logits_launch(h, "jss_step_logits", logits_dev, ld, seed, step_index, actions_out_dev, log_prob_out_dev, a)))
        return rc;
    return launch_all(h, a, (cudaStream_t)stream);
}

int jss_step_logits_record(jss_t *h, const float *logits_dev, int64_t ld, uint64_t seed, uint64_t step_index,
                           int32_t *actions_out_dev, float *log_prob_out_dev, float *obs_out_dev, uint8_t *mask_out_dev,
                           int32_t *scalars_out_dev, void *stream) {
    const char *what = "jss_step_logits_record";
    int rc = check_ready(h, stream);
    if (rc) return rc;
    JssLaunch a;
    if ((rc = logits_launch(h, what, logits_dev, ld, seed, step_index, actions_out_dev, log_prob_out_dev, a))) return rc;
    return launch_record(h, what, obs_out_dev, mask_out_dev, scalars_out_dev, a, (cudaStream_t)stream);
}

int jss_step_greedy(jss_t *h, const float *scores_dev, int64_t ld, double epsilon, uint64_t seed, uint64_t step_index,
                    int32_t *actions_out_dev, float *log_prob_out_dev, void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    JssLaunch a;
    if ((rc = greedy_launch(h, "jss_step_greedy", scores_dev, ld, epsilon, seed, step_index, actions_out_dev,
                            log_prob_out_dev, a)))
        return rc;
    return launch_all(h, a, (cudaStream_t)stream);
}

int jss_step_greedy_record(jss_t *h, const float *scores_dev, int64_t ld, double epsilon, uint64_t seed,
                           uint64_t step_index, int32_t *actions_out_dev, float *log_prob_out_dev, float *obs_out_dev,
                           uint8_t *mask_out_dev, int32_t *scalars_out_dev, void *stream) {
    const char *what = "jss_step_greedy_record";
    int rc = check_ready(h, stream);
    if (rc) return rc;
    JssLaunch a;
    if ((rc = greedy_launch(h, what, scores_dev, ld, epsilon, seed, step_index, actions_out_dev, log_prob_out_dev, a)))
        return rc;
    return launch_record(h, what, obs_out_dev, mask_out_dev, scalars_out_dev, a, (cudaStream_t)stream);
}

int jss_refresh_obs(jss_t *h, void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    return refresh_obs(h, (cudaStream_t)stream);
}

int jss_policy(jss_t *h, int rule, int coin_mode, uint64_t seed, uint64_t step_index, int32_t *actions_dev,
               void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    if (bad_ptr(actions_dev) || !valid_rule_coin(rule, coin_mode))
        return fail(h, JSS_ERR_INVALID, "jss_policy: bad arguments (rule %d, coin %d)", rule, coin_mode);
    JssLaunch a{};
    a.mode = JSS_MODE_POLICY;
    a.rule = rule; a.coin_mode = coin_mode; a.seed = seed; a.step_index = step_index; a.cr_factor = h->cr_factor;
    a.actions_out = actions_dev;
    return launch_all(h, a, (cudaStream_t)stream);
}

int jss_rollout(jss_t *h, int rule, uint64_t seed, uint64_t step_index, int n_steps, int write_obs, void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    if (!valid_rule_coin(rule, JSS_COIN_DEVICE) || n_steps < 0)
        return fail(h, JSS_ERR_INVALID, "jss_rollout: bad arguments (rule %d, n_steps %d)", rule, n_steps);
    JssLaunch a{};
    a.mode = JSS_MODE_ROLLOUT;
    a.rule = rule; a.coin_mode = JSS_COIN_DEVICE; a.seed = seed; a.step_index = step_index; a.cr_factor = h->cr_factor;
    a.n_steps = n_steps; a.write_obs = write_obs;
    return launch_all(h, a, (cudaStream_t)stream);
}

int jss_rollout_traj(jss_t *h, int rule, uint64_t seed, uint64_t step_index, int n_steps, float *traj_obs,
                     uint8_t *traj_mask, int32_t *traj_scalars, int32_t *traj_actions, void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    if (!valid_rule_coin(rule, JSS_COIN_DEVICE) || n_steps < 0 || !traj_obs || !traj_mask || !traj_scalars)
        return fail(h, JSS_ERR_INVALID, "jss_rollout_traj: bad arguments (rule %d, n_steps %d)", rule, n_steps);
    if ((int64_t)n_steps * h->n_envs >= INT32_MAX)
        return fail(h, JSS_ERR_UNSUPPORTED, "jss_rollout_traj: n_steps * n_envs must stay below 2^31");
    JssLaunch a{};
    a.mode = JSS_MODE_ROLLOUT;
    a.rule = rule; a.coin_mode = JSS_COIN_DEVICE; a.seed = seed; a.step_index = step_index; a.cr_factor = h->cr_factor;
    a.n_steps = n_steps; a.write_obs = 1;
    a.traj_obs = traj_obs; a.traj_mask = traj_mask; a.traj_scalars = traj_scalars; a.traj_actions = traj_actions;
    return launch_all(h, a, (cudaStream_t)stream);
}

int jss_rollout_priority(jss_t *h, const float *prio_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op, int n_steps,
                         void *stream) {
    const char *who = "jss_rollout_priority";
    int rc = check_ready(h, stream);
    if (rc) return rc;
    JssLaunch a{};
    if ((rc = table_arg(h, who, prio_dev, ld_env, ld_job, ld_op, a.table))) return rc;
    if (n_steps < 0) return fail(h, JSS_ERR_INVALID, "%s: bad arguments (n_steps %d >= 0)", who, n_steps);
    if (n_steps == 0) return JSS_OK;
    a.mode = JSS_MODE_PRIORITY;
    a.n_steps = n_steps;
    return launch_all(h, a, (cudaStream_t)stream);
}

namespace {

// the entropy forms take their sibling's arguments and checks, then their own outputs (ent)
int entropy_out_arg(jss_t *h, const char *who, bool ent, float *entropy_out) {
    if (ent && bad_ptr(entropy_out))
        return fail(h, JSS_ERR_INVALID, "%s: bad arguments (entropy_out %p must be non-NULL and 4-byte aligned)", who,
                    (void *)entropy_out);
    return JSS_OK;
}

int entropy_weights_arg(jss_t *h, const char *who, bool ent, const float *entropy_weights) {
    if (ent && bad_ptr(entropy_weights))
        return fail(h, JSS_ERR_INVALID, "%s: bad arguments (entropy_weights %p must be non-NULL and 4-byte aligned)",
                    who, (const void *)entropy_weights);
    return JSS_OK;
}

int rollout_priority_sample(jss_t *h, const char *who, bool ent, const float *logits_dev, int64_t ld_env,
                            int64_t ld_job, int64_t ld_op, uint64_t seed, uint64_t step_index, int n_steps,
                            float *log_prob_out_dev, float *entropy_out_dev, float *grad_out_dev,
                            float *entropy_grad_out_dev, void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    JssLaunch a{};
    if ((rc = table_arg(h, who, logits_dev, ld_env, ld_job, ld_op, a.table))) return rc;
    if (bad_ptr(log_prob_out_dev) || ((uintptr_t)grad_out_dev & 3u) || n_steps < 0)
        return fail(h, JSS_ERR_INVALID, "%s: bad arguments (log_prob_out %p must be non-NULL, it and grad_out %p "
                    "4-byte aligned, n_steps %d >= 0)", who, (void *)log_prob_out_dev, (void *)grad_out_dev, n_steps);
    if ((rc = entropy_out_arg(h, who, ent, entropy_out_dev))) return rc;
    if ((uintptr_t)entropy_grad_out_dev & 3u)
        return fail(h, JSS_ERR_INVALID, "%s: bad arguments (entropy_grad_out %p must be 4-byte aligned)", who,
                    (void *)entropy_grad_out_dev);
    if (n_steps == 0) return JSS_OK;
    a.mode = ent ? JSS_MODE_PRIORITY_SAMPLE_ENT : JSS_MODE_PRIORITY_SAMPLE;
    a.seed_folded = jss_fold32(seed);                    // jss_hash3 reads the seed only through its fold
    a.sample_counter = step_index;
    a.n_steps = n_steps;
    a.log_prob_out = log_prob_out_dev;
    a.grad_out = grad_out_dev;
    a.entropy_out = entropy_out_dev;
    a.entropy_grad_out = entropy_grad_out_dev;
    return launch_all(h, a, (cudaStream_t)stream);
}

}  // namespace

int jss_rollout_priority_sample(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                                uint64_t seed, uint64_t step_index, int n_steps, float *log_prob_out_dev,
                                float *grad_out_dev, void *stream) {
    return rollout_priority_sample(h, "jss_rollout_priority_sample", false, logits_dev, ld_env, ld_job, ld_op, seed,
                                   step_index, n_steps, log_prob_out_dev, nullptr, grad_out_dev, nullptr, stream);
}

int jss_rollout_priority_sample_entropy(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job,
                                        int64_t ld_op, uint64_t seed, uint64_t step_index, int n_steps,
                                        float *log_prob_out_dev, float *entropy_out_dev, float *grad_out_dev,
                                        float *entropy_grad_out_dev, void *stream) {
    return rollout_priority_sample(h, "jss_rollout_priority_sample_entropy", true, logits_dev, ld_env, ld_job, ld_op,
                                   seed, step_index, n_steps, log_prob_out_dev, entropy_out_dev, grad_out_dev,
                                   entropy_grad_out_dev, stream);
}

int jss_lookahead(jss_t *h, int rule, int coin_mode, uint64_t seed, uint64_t step_index, int32_t *makespan_out_dev,
                  int64_t ld, void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    if (!valid_rule_coin(rule, coin_mode) || bad_ptr(makespan_out_dev) || ld < (int64_t)h->p.jobs_max + 1)
        return fail(h, JSS_ERR_INVALID, "jss_lookahead: bad arguments (rule %d, coin %d, makespan_out %p must be "
                    "4-byte aligned, ld %lld >= jobs_max + 1 = %d)", rule, coin_mode, (void *)makespan_out_dev,
                    (long long)ld, h->p.jobs_max + 1);
    JssLaunch a{};
    a.mode = JSS_MODE_LOOKAHEAD;
    a.rule = rule; a.coin_mode = coin_mode; a.seed = seed; a.step_index = step_index; a.cr_factor = h->cr_factor;
    a.values_out = makespan_out_dev;
    a.out_ld = ld;
    return launch_all(h, a, (cudaStream_t)stream);
}

int jss_lookahead_priority(jss_t *h, const float *prio_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                           int32_t *makespan_out_dev, int64_t ld, void *stream) {
    const char *who = "jss_lookahead_priority";
    int rc = check_ready(h, stream);
    if (rc) return rc;
    JssLaunch a{};
    if ((rc = table_arg(h, who, prio_dev, ld_env, ld_job, ld_op, a.table))) return rc;
    if (bad_ptr(makespan_out_dev) || ld < (int64_t)h->p.jobs_max + 1)
        return fail(h, JSS_ERR_INVALID, "%s: bad arguments (makespan_out %p must be non-NULL and 4-byte aligned, ld "
                    "%lld >= jobs_max + 1 = %d)", who, (void *)makespan_out_dev, (long long)ld, h->p.jobs_max + 1);
    a.mode = JSS_MODE_LOOKAHEAD_PRIORITY;
    a.values_out = makespan_out_dev;
    a.out_ld = ld;
    return launch_all(h, a, (cudaStream_t)stream);
}

namespace {

// a.beam_trace for a (stochastic) beam search of width W that writes orders: W backpointers per round (at most
// jobs_max * machines_max rounds) for each CTA of the largest grid, owned by the handle and grown as needed
int beam_trace(jss_t *h, JssLaunch &a) {
    JssLaunch g = a;
    size_t smem = 0;
    mode_layout(h, g, smem);
    int grid_max = 0;
    for (int c = 0; c < JSS_LANE_CLASSES; c++) {
        g.tile_begin = h->class_tiles[c][0];
        g.tile_end = h->class_tiles[c][1];
        if (g.tile_end <= g.tile_begin) continue;
        int grid = 0;
        if (int rc = mode_grid(h, g, c, smem, grid)) return rc;
        grid_max = std::max(grid_max, grid);
    }
    const size_t need = (size_t)grid_max * a.beam_width * h->p.jobs_max * h->p.machines_max * sizeof(uint16_t);
    if (need > h->beam_trace_bytes) {
        if (h->beam_trace) {                             // cudaFree waits for the launches that may still use it
            JSS_CUDA(h, cudaFree(h->beam_trace));
            h->beam_trace = nullptr;
            h->beam_trace_bytes = 0;
        }
        void *ptr = nullptr;
        JSS_CUDA(h, cudaMalloc(&ptr, need));
        h->beam_trace = static_cast<uint16_t *>(ptr);
        h->beam_trace_bytes = need;
    }
    a.beam_trace = h->beam_trace;
    return JSS_OK;
}

// the arguments jss_sample_episodes and its replays share: the table as jss_rollout_priority_sample takes it, the seed
// and counter; k and ld where the call has them (has_k)
int sample_episodes_args(jss_t *h, const char *who, const float *logits, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                         uint64_t seed, uint64_t step_index, bool has_k, int64_t k, int64_t ld, JssLaunch &a) {
    if (int rc = table_arg(h, who, logits, ld_env, ld_job, ld_op, a.table)) return rc;
    if (has_k) {
        const uint64_t bound = 2ull * (uint64_t)h->p.jobs_max * (uint64_t)h->p.machines_max + 1;
        if (k < 1 || ld < k || (uint64_t)k > UINT64_MAX / bound)
            return fail(h, JSS_ERR_INVALID, "%s: bad arguments (k %lld >= 1 with k * (2 * J * M + 1) below 2^64, "
                        "ld %lld >= k)", who, (long long)k, (long long)ld);
        if (k > INT32_MAX)
            return fail(h, JSS_ERR_UNSUPPORTED, "%s: k must stay below 2^31", who);
        a.n_samples = (int)k;
        a.out_ld = ld;
    }
    a.seed_folded = jss_fold32(seed);                    // jss_hash3 reads the seed only through its fold
    a.sample_counter = step_index;
    return JSS_OK;
}

int sample_episodes(jss_t *h, const char *who, bool ent, const float *logits_dev, int64_t ld_env, int64_t ld_job,
                    int64_t ld_op, uint64_t seed, uint64_t step_index, int64_t k, int32_t *makespan_out_dev,
                    float *log_prob_out_dev, float *entropy_out_dev, int64_t ld, void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    if (bad_ptr(makespan_out_dev) || bad_ptr(log_prob_out_dev))
        return fail(h, JSS_ERR_INVALID, "%s: bad arguments (makespan_out %p and log_prob_out %p must be 4-byte "
                    "aligned)", who, (void *)makespan_out_dev, (void *)log_prob_out_dev);
    if ((rc = entropy_out_arg(h, who, ent, entropy_out_dev))) return rc;
    JssLaunch a{};
    a.mode = ent ? JSS_MODE_SAMPLE_EPISODES_ENT : JSS_MODE_SAMPLE_EPISODES;
    if ((rc = sample_episodes_args(h, who, logits_dev, ld_env, ld_job, ld_op, seed, step_index, true, k, ld, a)))
        return rc;
    a.makespan_out = makespan_out_dev;
    a.log_prob_out = log_prob_out_dev;
    a.entropy_out = entropy_out_dev;
    return launch_all(h, a, (cudaStream_t)stream);
}

int sample_episodes_grad(jss_t *h, const char *who, bool ent, const float *logits_dev, int64_t ld_env, int64_t ld_job,
                         int64_t ld_op, uint64_t seed, uint64_t step_index, int64_t k, const float *weights_dev,
                         const float *entropy_weights_dev, int64_t ld, int split, float *grad_out_dev, void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    if (bad_ptr(weights_dev) || bad_ptr(grad_out_dev) || split < 1 || split > k)
        return fail(h, JSS_ERR_INVALID, "%s: bad arguments (weights %p and grad_out %p must be 4-byte aligned, "
                    "1 <= split %d <= k %lld)", who, (const void *)weights_dev, (void *)grad_out_dev, split,
                    (long long)k);
    if ((rc = entropy_weights_arg(h, who, ent, entropy_weights_dev))) return rc;
    if ((int64_t)h->n_tiles * split > INT32_MAX)
        return fail(h, JSS_ERR_UNSUPPORTED, "%s: split * tiles must stay below 2^31", who);
    JssLaunch a{};
    a.mode = ent ? JSS_MODE_SAMPLE_EPISODES_ENT_GRAD : JSS_MODE_SAMPLE_EPISODES_GRAD;
    if ((rc = sample_episodes_args(h, who, logits_dev, ld_env, ld_job, ld_op, seed, step_index, true, k, ld, a)))
        return rc;
    a.weights = weights_dev;
    a.entropy_weights = entropy_weights_dev;
    a.split = split;
    a.grad_out = grad_out_dev;
    return launch_all(h, a, (cudaStream_t)stream);
}

}  // namespace

int jss_sample_episodes(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                        uint64_t seed, uint64_t step_index, int64_t k, int32_t *makespan_out_dev,
                        float *log_prob_out_dev, int64_t ld, void *stream) {
    return sample_episodes(h, "jss_sample_episodes", false, logits_dev, ld_env, ld_job, ld_op, seed, step_index, k,
                           makespan_out_dev, log_prob_out_dev, nullptr, ld, stream);
}

int jss_sample_episodes_entropy(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                                uint64_t seed, uint64_t step_index, int64_t k, int32_t *makespan_out_dev,
                                float *log_prob_out_dev, float *entropy_out_dev, int64_t ld, void *stream) {
    return sample_episodes(h, "jss_sample_episodes_entropy", true, logits_dev, ld_env, ld_job, ld_op, seed, step_index,
                           k, makespan_out_dev, log_prob_out_dev, entropy_out_dev, ld, stream);
}

int jss_sample_episodes_grad(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                             uint64_t seed, uint64_t step_index, int64_t k, const float *weights_dev, int64_t ld,
                             int split, float *grad_out_dev, void *stream) {
    return sample_episodes_grad(h, "jss_sample_episodes_grad", false, logits_dev, ld_env, ld_job, ld_op, seed,
                                step_index, k, weights_dev, nullptr, ld, split, grad_out_dev, stream);
}

int jss_sample_episodes_entropy_grad(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                                     uint64_t seed, uint64_t step_index, int64_t k, const float *weights_dev,
                                     const float *entropy_weights_dev, int64_t ld, int split, float *grad_out_dev,
                                     void *stream) {
    return sample_episodes_grad(h, "jss_sample_episodes_entropy_grad", true, logits_dev, ld_env, ld_job, ld_op, seed,
                                step_index, k, weights_dev, entropy_weights_dev, ld, split, grad_out_dev, stream);
}

int jss_sample_episodes_solution(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                                 uint64_t seed, uint64_t step_index, const int32_t *sample_dev,
                                 int32_t *solution_out_dev, void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    const char *who = "jss_sample_episodes_solution";
    if (bad_ptr(sample_dev) || bad_ptr(solution_out_dev))
        return fail(h, JSS_ERR_INVALID, "%s: bad arguments (sample %p and solution_out %p must be 4-byte aligned)",
                    who, (const void *)sample_dev, (void *)solution_out_dev);
    JssLaunch a{};
    a.mode = JSS_MODE_SAMPLE_EPISODES_SOLUTION;
    if ((rc = sample_episodes_args(h, who, logits_dev, ld_env, ld_job, ld_op, seed, step_index, false, 0, 0, a)))
        return rc;
    a.sample_in = sample_dev;
    a.solution_out = solution_out_dev;
    a.split = 1;
    return launch_all(h, a, (cudaStream_t)stream);
}

int jss_lookahead_sample(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                         uint64_t seed, uint64_t step_index, int64_t k, int32_t *makespan_out_dev, int64_t ld,
                         void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    const char *who = "jss_lookahead_sample";
    JssLaunch a{};
    a.mode = JSS_MODE_LOOKAHEAD_SAMPLE;
    if ((rc = sample_episodes_args(h, who, logits_dev, ld_env, ld_job, ld_op, seed, step_index, true, k, ld, a)))
        return rc;
    const int64_t row = (int64_t)(h->p.jobs_max + 1) * k;   // k < 2^31 here
    if (bad_ptr(makespan_out_dev) || ld < row)
        return fail(h, JSS_ERR_INVALID, "%s: bad arguments (makespan_out %p must be non-NULL and 4-byte aligned, ld "
                    "%lld >= (jobs_max + 1) * k = %lld)", who, (void *)makespan_out_dev, (long long)ld,
                    (long long)row);
    // a tile's split reaches (jobs_max + 1) k at most: its work items, and an env's pairs, stay below 2^31
    if ((int64_t)h->n_tiles * row > INT32_MAX)
        return fail(h, JSS_ERR_UNSUPPORTED, "%s: tiles * (jobs_max + 1) * k must stay below 2^31", who);
    a.values_out = makespan_out_dev;
    return launch_all(h, a, (cudaStream_t)stream);
}

int jss_beam_search(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op, int width,
                    int32_t *makespan_out_dev, float *score_out_dev, int64_t ld, int32_t *order_out_dev, void *stream) {
    const char *who = "jss_beam_search";
    int rc = check_ready(h, stream);
    if (rc) return rc;
    JssLaunch a{};
    if ((rc = table_arg(h, who, logits_dev, ld_env, ld_job, ld_op, a.table))) return rc;
    if (bad_ptr(makespan_out_dev) || bad_ptr(score_out_dev) || ((uintptr_t)order_out_dev & 3u) || width < 1 ||
        width > JSS_MAX_BEAM_WIDTH || ld < width)
        return fail(h, JSS_ERR_INVALID, "%s: bad arguments (makespan_out %p and score_out %p must be non-NULL, they "
                    "and order_out %p 4-byte aligned, 1 <= width %d <= %d, ld %lld >= width)", who,
                    (void *)makespan_out_dev, (void *)score_out_dev, (void *)order_out_dev, width, JSS_MAX_BEAM_WIDTH,
                    (long long)ld);
    a.mode = JSS_MODE_BEAM_SEARCH;
    a.beam_width = width;
    a.makespan_out = makespan_out_dev;
    a.score_out = score_out_dev;
    a.out_ld = ld;
    a.order_out = order_out_dev;
    if (order_out_dev && (rc = beam_trace(h, a))) return rc;
    return launch_all(h, a, (cudaStream_t)stream);
}

int jss_sample_without_replacement(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                                   uint64_t seed, uint64_t step_index, int width, int32_t *makespan_out_dev,
                                   float *log_prob_out_dev, float *key_out_dev, int64_t ld, int32_t *order_out_dev,
                                   void *stream) {
    const char *who = "jss_sample_without_replacement";
    int rc = check_ready(h, stream);
    if (rc) return rc;
    JssLaunch a{};
    if ((rc = table_arg(h, who, logits_dev, ld_env, ld_job, ld_op, a.table))) return rc;
    if (bad_ptr(makespan_out_dev) || bad_ptr(log_prob_out_dev) || bad_ptr(key_out_dev) ||
        ((uintptr_t)order_out_dev & 3u) || width < 1 || width > JSS_MAX_BEAM_WIDTH || ld < width)
        return fail(h, JSS_ERR_INVALID, "%s: bad arguments (makespan_out %p, log_prob_out %p and key_out %p must be "
                    "non-NULL, they and order_out %p 4-byte aligned, 1 <= width %d <= %d, ld %lld >= width)", who,
                    (void *)makespan_out_dev, (void *)log_prob_out_dev, (void *)key_out_dev, (void *)order_out_dev,
                    width, JSS_MAX_BEAM_WIDTH, (long long)ld);
    a.mode = JSS_MODE_SWOR;
    a.seed_folded = jss_fold32(seed);                    // jss_hash3 reads the seed only through its fold
    a.sample_counter = step_index;
    a.beam_width = width;
    a.makespan_out = makespan_out_dev;
    a.log_prob_out = log_prob_out_dev;
    a.key_out = key_out_dev;
    a.out_ld = ld;
    a.order_out = order_out_dev;
    if (order_out_dev && (rc = beam_trace(h, a))) return rc;
    return launch_all(h, a, (cudaStream_t)stream);
}

namespace {

// jss_beam_step's group records for width W, built once per handle and width: per group [g, instance, the W slots'
// block offsets in 16-byte units] (blocks are in tile order, and a group need not align with tiles), grouped by lane
// class and, within one, by instance, so that a CTA restages the instance tables rarely.  Leaves `out` null with the
// reason in the handle's error (after `who`) if the width does not divide N or a group mixes instances.
int beam_groups(jss_t *h, const char *who, int W, const jss_handle::BeamGroups *&out) {
    out = nullptr;
    auto it = h->beam_groups.find(W);
    if (it == h->beam_groups.end()) {
        jss_handle::BeamGroups bg;
        const int N = h->n_envs, G = N / W;
        if (N % W) {
            bg.err = "width " + std::to_string(W) + " does not divide the " + std::to_string(N) + " envs";
        } else {
            for (int g = 0; g < G && bg.err.empty(); g++)
                for (int b = 1; b < W; b++)
                    if (h->env_inst[g * W + b] != h->env_inst[g * W]) {
                        bg.err = "group " + std::to_string(g) + " (envs " + std::to_string(g * W) + " .. " +
                                 std::to_string(g * W + W - 1) + ") mixes instances";
                        break;
                    }
        }
        if (bg.err.empty()) {
            std::vector<int32_t> grp(G);
            for (int g = 0; g < G; g++) grp[g] = g;
            const auto cls = [&](int g) { return jss_lane_class(h->insts[h->env_inst[g * W]].J); };
            std::stable_sort(grp.begin(), grp.end(), [&](int x, int y) {
                if (cls(x) != cls(y)) return cls(x) < cls(y);
                return h->env_inst[x * W] < h->env_inst[y * W];
            });
            std::vector<int32_t> rec((size_t)G * (W + 2));
            for (int r = 0; r < G; r++) {
                const int g = grp[r], c = cls(g);
                int32_t *q = rec.data() + (size_t)r * (W + 2);
                q[0] = g;
                q[1] = h->env_inst[g * W];
                for (int b = 0; b < W; b++) q[2 + b] = (int32_t)h->env_off16[g * W + b];
                if (r == 0 || cls(grp[r - 1]) != c) bg.ranges[c][0] = r;
                bg.ranges[c][1] = r + 1;
            }
            if (int rc = dev_alloc(h, &bg.dev, rec.size(), false)) return rc;
            JSS_CUDA(h, cudaMemcpy(bg.dev, rec.data(), rec.size() * 4, cudaMemcpyHostToDevice));
            JSS_CUDA(h, cudaStreamSynchronize(nullptr));   // a caller's non-blocking stream does not wait for it
        }
        it = h->beam_groups.emplace(W, bg).first;
    }
    if (!it->second.err.empty()) return fail(h, JSS_ERR_INVALID, "%s: %s", who, it->second.err.c_str());
    out = &it->second;
    return JSS_OK;
}

// jss_beam_step and jss_stochastic_beam_step (key_dev non-NULL): the checks and the group records
int beam_step_launch(jss_t *h, const char *who, const float *logits_dev, int64_t ld, int width, uint64_t seed,
                     uint64_t step_index, float *score_dev, float *key_dev, int32_t *parent_out_dev,
                     int32_t *action_out_dev, int32_t *bad_out_dev, void *stream) {
    const bool swor = key_dev != nullptr;
    if (bad_ptr(logits_dev) || bad_ptr(score_dev) || bad_ptr(parent_out_dev) || bad_ptr(action_out_dev) ||
        bad_ptr(bad_out_dev) || width < 1 || width > JSS_MAX_BEAM_WIDTH || ld < (int64_t)h->p.jobs_max + 1)
        return fail(h, JSS_ERR_INVALID, "%s: bad arguments (logits %p, score %p, parent_out %p, action_out "
                    "%p and bad_out %p must be non-NULL and 4-byte aligned, 1 <= width %d <= %d, ld %lld >= jobs_max + 1 "
                    "= %d)", who, (const void *)logits_dev, (void *)score_dev, (void *)parent_out_dev,
                    (void *)action_out_dev, (void *)bad_out_dev, width, JSS_MAX_BEAM_WIDTH, (long long)ld,
                    h->p.jobs_max + 1);
    if (swor && h->env_id_base % (uint64_t)width)
        return fail(h, JSS_ERR_INVALID, "%s: env_id_base %llu is not a multiple of width %d (group ids are "
                    "env_id_base / width + g)", who, (unsigned long long)h->env_id_base, width);
    int rc;
    const jss_handle::BeamGroups *bg = nullptr;
    if ((rc = beam_groups(h, who, width, bg))) return rc;
    JssLaunch a{};
    a.mode = swor ? JSS_MODE_STOCHASTIC_BEAM_STEP : JSS_MODE_BEAM_STEP;
    a.beam_width = width;
    a.beam_groups = bg->dev;
    a.rows = logits_dev;
    a.rows_ld = ld;
    a.score_io = score_dev;
    a.parent_out = parent_out_dev;
    a.job_out = action_out_dev;
    a.bad_out = bad_out_dev;
    if (swor) {
        a.key_io = key_dev;
        a.seed_folded = jss_fold32(seed);                // jss_hash3 reads the seed only through its fold
        a.sample_counter = step_index;
    }
    return launch_all(h, a, (cudaStream_t)stream, bg->ranges);
}

}  // namespace

int jss_beam_step(jss_t *h, const float *logits_dev, int64_t ld, int width, float *score_dev, int32_t *parent_out_dev,
                  int32_t *action_out_dev, int32_t *bad_out_dev, void *stream) {
    const int rc = check_ready(h, stream);
    if (rc) return rc;
    return beam_step_launch(h, "jss_beam_step", logits_dev, ld, width, 0, 0, score_dev, nullptr, parent_out_dev,
                            action_out_dev, bad_out_dev, stream);
}

int jss_stochastic_beam_step(jss_t *h, const float *logits_dev, int64_t ld, int width, uint64_t seed,
                             uint64_t step_index, float *score_dev, float *key_dev, int32_t *parent_out_dev,
                             int32_t *action_out_dev, int32_t *bad_out_dev, void *stream) {
    const int rc = check_ready(h, stream);
    if (rc) return rc;
    if (bad_ptr(key_dev))
        return fail(h, JSS_ERR_INVALID, "jss_stochastic_beam_step: bad arguments (key %p must be non-NULL and 4-byte "
                    "aligned)", (void *)key_dev);
    return beam_step_launch(h, "jss_stochastic_beam_step", logits_dev, ld, width, seed, step_index, score_dev, key_dev,
                            parent_out_dev, action_out_dev, bad_out_dev, stream);
}

namespace {

// K operation orders per env, and the row stride of the per-order outputs
int orders_arg(jss_t *h, const char *who, const int32_t *order, int64_t k, int64_t ld, JssLaunch &a) {
    if (bad_ptr(order) || k < 1 || ld < k)
        return fail(h, JSS_ERR_INVALID, "%s: bad arguments (order %p must be non-NULL and 4-byte aligned, k %lld >= 1, "
                    "ld %lld >= k)", who, (const void *)order, (long long)k, (long long)ld);
    if (k > INT32_MAX)
        return fail(h, JSS_ERR_UNSUPPORTED, "%s: k must stay below 2^31", who);
    a.order_in = order;
    a.n_samples = (int)k;
    a.out_ld = ld;
    return JSS_OK;
}

// the arguments jss_order_log_prob and its gradient share: the table as jss_rollout_priority_sample takes it, k orders
// per env, and ld
int order_log_prob_args(jss_t *h, const char *who, const float *logits, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                        const int32_t *order, int64_t k, int64_t ld, JssLaunch &a) {
    if (int rc = table_arg(h, who, logits, ld_env, ld_job, ld_op, a.table)) return rc;
    return orders_arg(h, who, order, k, ld, a);
}

int order_log_prob(jss_t *h, const char *who, bool ent, const float *logits_dev, int64_t ld_env, int64_t ld_job,
                   int64_t ld_op, const int32_t *order_dev, int64_t k, int32_t *makespan_out_dev,
                   float *log_prob_out_dev, float *entropy_out_dev, int64_t ld, void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    if (bad_ptr(makespan_out_dev) || bad_ptr(log_prob_out_dev))
        return fail(h, JSS_ERR_INVALID, "%s: bad arguments (makespan_out %p and log_prob_out %p must be non-NULL and "
                    "4-byte aligned)", who, (void *)makespan_out_dev, (void *)log_prob_out_dev);
    if ((rc = entropy_out_arg(h, who, ent, entropy_out_dev))) return rc;
    JssLaunch a{};
    a.mode = ent ? JSS_MODE_ORDER_LOG_PROB_ENT : JSS_MODE_ORDER_LOG_PROB;
    if ((rc = order_log_prob_args(h, who, logits_dev, ld_env, ld_job, ld_op, order_dev, k, ld, a))) return rc;
    a.makespan_out = makespan_out_dev;
    a.log_prob_out = log_prob_out_dev;
    a.entropy_out = entropy_out_dev;
    return launch_all(h, a, (cudaStream_t)stream);
}

int order_log_prob_grad(jss_t *h, const char *who, bool ent, const float *logits_dev, int64_t ld_env, int64_t ld_job,
                        int64_t ld_op, const int32_t *order_dev, int64_t k, const float *weights_dev,
                        const float *entropy_weights_dev, int64_t ld, int split, float *grad_out_dev, void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    if (bad_ptr(weights_dev) || bad_ptr(grad_out_dev) || split < 1 || split > k)
        return fail(h, JSS_ERR_INVALID, "%s: bad arguments (weights %p and grad_out %p must be non-NULL and 4-byte "
                    "aligned, 1 <= split %d <= k %lld)", who, (const void *)weights_dev, (void *)grad_out_dev, split,
                    (long long)k);
    if ((rc = entropy_weights_arg(h, who, ent, entropy_weights_dev))) return rc;
    if ((int64_t)h->n_tiles * split > INT32_MAX)
        return fail(h, JSS_ERR_UNSUPPORTED, "%s: split * tiles must stay below 2^31", who);
    JssLaunch a{};
    a.mode = ent ? JSS_MODE_ORDER_LOG_PROB_ENT_GRAD : JSS_MODE_ORDER_LOG_PROB_GRAD;
    if ((rc = order_log_prob_args(h, who, logits_dev, ld_env, ld_job, ld_op, order_dev, k, ld, a))) return rc;
    a.weights = weights_dev;
    a.entropy_weights = entropy_weights_dev;
    a.split = split;
    a.grad_out = grad_out_dev;
    return launch_all(h, a, (cudaStream_t)stream);
}

}  // namespace

int jss_order_log_prob(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                       const int32_t *order_dev, int64_t k, int32_t *makespan_out_dev, float *log_prob_out_dev,
                       int64_t ld, void *stream) {
    return order_log_prob(h, "jss_order_log_prob", false, logits_dev, ld_env, ld_job, ld_op, order_dev, k,
                          makespan_out_dev, log_prob_out_dev, nullptr, ld, stream);
}

int jss_order_log_prob_entropy(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                               const int32_t *order_dev, int64_t k, int32_t *makespan_out_dev, float *log_prob_out_dev,
                               float *entropy_out_dev, int64_t ld, void *stream) {
    return order_log_prob(h, "jss_order_log_prob_entropy", true, logits_dev, ld_env, ld_job, ld_op, order_dev, k,
                          makespan_out_dev, log_prob_out_dev, entropy_out_dev, ld, stream);
}

int jss_order_log_prob_grad(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                            const int32_t *order_dev, int64_t k, const float *weights_dev, int64_t ld, int split,
                            float *grad_out_dev, void *stream) {
    return order_log_prob_grad(h, "jss_order_log_prob_grad", false, logits_dev, ld_env, ld_job, ld_op, order_dev, k,
                               weights_dev, nullptr, ld, split, grad_out_dev, stream);
}

int jss_order_log_prob_entropy_grad(jss_t *h, const float *logits_dev, int64_t ld_env, int64_t ld_job, int64_t ld_op,
                                    const int32_t *order_dev, int64_t k, const float *weights_dev,
                                    const float *entropy_weights_dev, int64_t ld, int split, float *grad_out_dev,
                                    void *stream) {
    return order_log_prob_grad(h, "jss_order_log_prob_entropy_grad", true, logits_dev, ld_env, ld_job, ld_op,
                               order_dev, k, weights_dev, entropy_weights_dev, ld, split, grad_out_dev, stream);
}

int jss_improve_orders(jss_t *h, const int32_t *order_dev, int64_t k, int max_moves, int32_t *order_out_dev,
                       int32_t *makespan_out_dev, int32_t *start_makespan_out_dev, int32_t *moves_out_dev, int64_t ld,
                       void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    const char *who = "jss_improve_orders";
    if (bad_ptr(order_out_dev) || bad_ptr(makespan_out_dev) || bad_ptr(start_makespan_out_dev) ||
        bad_ptr(moves_out_dev) || max_moves < 0)
        return fail(h, JSS_ERR_INVALID, "%s: bad arguments (order_out %p, makespan_out %p, start_makespan_out %p and "
                    "moves_out %p must be non-NULL and 4-byte aligned, max_moves %d >= 0)", who, (void *)order_out_dev,
                    (void *)makespan_out_dev, (void *)start_makespan_out_dev, (void *)moves_out_dev, max_moves);
    JssLaunch a{};
    if ((rc = orders_arg(h, who, order_dev, k, ld, a))) return rc;
    // the byte ranges the call reads or writes; only order_out == order may share one
    const uint64_t N = (uint64_t)h->n_envs, ords = N * (uint64_t)k * h->p.jobs_max * h->p.machines_max * 4,
                   rows = ((N - 1) * (uint64_t)ld + (uint64_t)k) * 4;
    const struct { const void *p; uint64_t bytes; } span[5] = {{order_dev, ords}, {order_out_dev, ords},
        {makespan_out_dev, rows}, {start_makespan_out_dev, rows}, {moves_out_dev, rows}};
    for (int x = 0; x < 5; x++)
        for (int y = x + 1; y < 5; y++) {
            const uintptr_t px = (uintptr_t)span[x].p, py = (uintptr_t)span[y].p;
            if (x == 0 && y == 1 && px == py) continue;  // in place
            if (px < py + span[y].bytes && py < px + span[x].bytes)
                return fail(h, JSS_ERR_INVALID, "%s: bad arguments (buffers %d and %d overlap; only order_out == order "
                            "may)", who, x, y);
        }
    a.mode = JSS_MODE_IMPROVE_ORDERS;
    a.max_moves = max_moves;
    a.order_out = order_out_dev;
    a.makespan_out = makespan_out_dev;
    a.start_out = start_makespan_out_dev;
    a.moves_out = moves_out_dev;
    return launch_all(h, a, (cudaStream_t)stream);
}

int jss_step_host(jss_t *h, const int32_t *actions_host, uint8_t *mask_host, float *obs_host,
                  int32_t *scalars_host, void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    if (!actions_host) return fail(h, JSS_ERR_INVALID, "jss_step_host: actions_host is NULL");
    cudaStream_t st = (cudaStream_t)stream;
    const JssParams &p = h->p;
    const size_t N = (size_t)p.n_envs;
    JSS_CUDA(h, cudaMemcpyAsync(h->dev_actions, actions_host, N * 4, cudaMemcpyHostToDevice, st));
    rc = jss_step(h, h->dev_actions, stream);
    if (rc) return rc;
    // contiguous DMA only: host rows keep the device pitches (mask rows: mask_stride bytes,
    // scalar records: 16 bytes) -- pitched 2-D copies of 65 536 tiny rows are several times slower
    if (mask_host)
        JSS_CUDA(h, cudaMemcpyAsync(mask_host, p.mask, N * p.mask_stride, cudaMemcpyDeviceToHost, st));
    if (obs_host)
        JSS_CUDA(h, cudaMemcpyAsync(obs_host, p.obs, N * p.jobs_max * 7 * 4, cudaMemcpyDeviceToHost, st));
    if (scalars_host) JSS_CUDA(h, cudaMemcpyAsync(scalars_host, p.scalars, N * 16, cudaMemcpyDeviceToHost, st));
    JSS_CUDA(h, cudaStreamSynchronize(st));
    return JSS_OK;
}

namespace {
// obs_host != NULL: envs [0, n_dma) ship their observation as fp32 rows by DMA (n_dma < 0: all of them);
// wire_host != NULL: envs [max(n_dma, 0), N) ship packed integer rows.
int host_step_begin_impl(jss_t *h, const int32_t *actions_host, uint8_t *mask_host, float *obs_host, uint8_t *wire_host,
                         int32_t *scalars_host, void *after_stream, int n_dma = -1) {
    int rc = check_ready(h);           // the pipeline orders itself: s_compute follows after_stream and itself
    if (rc) return rc;
    if (!actions_host) return fail(h, JSS_ERR_INVALID, "jss_host_step_begin: actions_host is NULL");
    const JssParams &p = h->p;
    const size_t N = (size_t)p.n_envs;
    const size_t n_fp32 = obs_host ? (n_dma < 0 ? N : std::min<size_t>((size_t)n_dma, N)) : 0;     // envs [0, n_fp32): fp32 by DMA
    const size_t obs_bytes = n_fp32 * p.jobs_max * 7 * 4;
    if (!h->pipe_ready) {
        JSS_CUDA(h, cudaStreamCreateWithFlags(&h->s_compute, cudaStreamNonBlocking));
        JSS_CUDA(h, cudaStreamCreateWithFlags(&h->s_copy, cudaStreamNonBlocking));
        JSS_CUDA(h, cudaEventCreateWithFlags(&h->ev_mask, cudaEventDisableTiming));
        JSS_CUDA(h, cudaEventCreateWithFlags(&h->ev_staged, cudaEventDisableTiming));
        JSS_CUDA(h, cudaEventCreateWithFlags(&h->ev_wire, cudaEventDisableTiming));
        for (int k = 0; k < 2; k++) {
            JSS_CUDA(h, cudaEventCreateWithFlags(&h->ev_obs[k], cudaEventDisableTiming));
            JSS_CUDA(h, cudaEventRecord(h->ev_obs[k], h->s_copy));
        }
        h->pipe_ready = true;
    }
    if (obs_host && !h->obs_staging && (rc = dev_alloc(h, &h->obs_staging, N * p.jobs_max * 7, false))) return rc;
    if (wire_host && !h->wire[0]) {
        h->wire_stride = jss_host_wire_stride(h);
        for (int k = 0; k < 2; k++)
            if ((rc = dev_alloc(h, &h->wire[k], N * (size_t)h->wire_stride))) return rc;
    }
    cudaStream_t sc = h->s_compute;
    // order the pipeline after whatever the caller enqueued on its own stream (reset, device-side steps ...)
    JSS_CUDA(h, cudaEventRecord(h->ev_staged, (cudaStream_t)after_stream));
    JSS_CUDA(h, cudaStreamWaitEvent(sc, h->ev_staged, 0));
    JSS_CUDA(h, cudaMemcpyAsync(h->dev_actions, actions_host, N * 4, cudaMemcpyHostToDevice, sc));
    rc = jss_step(h, h->dev_actions, (void *)sc);
    if (rc) return rc;
    // the small results first: a host policy only needs the mask.  If the host buffers are pinned
    // (device-mappable) the SMs write them directly; otherwise fall back to the copy engine.
    auto small_d2h = [&](void *dst_host, const void *src_dev, size_t bytes) -> int {
        void *mapped = nullptr;
        if ((bytes & 15) == 0 && cudaHostGetDevicePointer(&mapped, dst_host, 0) == cudaSuccess && mapped) {
            const size_t n16 = bytes / 16;
            const int blocks = (int)std::min<size_t>((n16 + 255) / 256, (size_t)h->sm_count * 8);
            JSS_LAUNCH(jss_copy16_kernel, blocks, 256, 0, sc, (uint4 *)mapped, (const uint4 *)src_dev, n16);
            JSS_CUDA(h, cudaGetLastError());
            h->launches += 1;
        } else {
            (void)cudaGetLastError();
            JSS_CUDA(h, cudaMemcpyAsync(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost, sc));
        }
        return JSS_OK;
    };
    if (mask_host && (rc = small_d2h(mask_host, p.mask, N * p.mask_stride))) return rc;
    if (scalars_host && (rc = small_d2h(scalars_host, p.scalars, N * 16))) return rc;
    JSS_CUDA(h, cudaEventRecord(h->ev_mask, sc));
    const int prev = h->pipe_cur;
    h->pipe_cur ^= 1;
    if (obs_bytes) {
        // observation: device-side staging copy (so the next step may overwrite real_obs), then the
        // 2.9 KB/env PCIe transfer on its own stream, overlapping the host policy and the next launch
        JSS_CUDA(h, cudaStreamWaitEvent(sc, h->ev_obs[prev], 0));      // previous D2H has drained the staging copy
        JSS_CUDA(h, cudaMemcpyAsync(h->obs_staging, p.obs, obs_bytes, cudaMemcpyDeviceToDevice, sc));
    }
    if (wire_host && n_fp32 < N) {
        // packed rows: 10 bytes per job instead of 28; two device buffers alternate, so this pack only has to wait
        // for the D2H that read the same buffer two begins ago
        JSS_CUDA(h, cudaStreamWaitEvent(sc, h->ev_obs[h->pipe_cur], 0));
        JssLaunch a{};
        a.mode = JSS_MODE_PACK;
        a.wire = h->wire[h->pipe_cur];
        a.wire_stride = (int32_t)h->wire_stride;
        if ((rc = launch_all(h, a, sc))) return rc;
    }
    // the copy stream never runs ahead of the step (also when nothing large is copied: ev_obs is what JSS_WAIT_OBS and
    // the stream-ordered entry points wait for)
    JSS_CUDA(h, cudaEventRecord(h->ev_staged, sc));
    JSS_CUDA(h, cudaStreamWaitEvent(h->s_copy, h->ev_staged, 0));
    if (wire_host && n_fp32 < N) {       // the packed rows first: the host has to expand them, the fp32 rows are final
        const size_t off = n_fp32 * (size_t)h->wire_stride;
        JSS_CUDA(h, cudaMemcpyAsync(wire_host + off, h->wire[h->pipe_cur] + off, (N - n_fp32) * (size_t)h->wire_stride,
                                    cudaMemcpyDeviceToHost, h->s_copy));
        JSS_CUDA(h, cudaEventRecord(h->ev_wire, h->s_copy));
    }
    if (obs_bytes)
        JSS_CUDA(h, cudaMemcpyAsync(obs_host, h->obs_staging, obs_bytes, cudaMemcpyDeviceToHost, h->s_copy));
    JSS_CUDA(h, cudaEventRecord(h->ev_obs[h->pipe_cur], h->s_copy));
    return JSS_OK;
}
}  // namespace

int jss_host_step_begin(jss_t *h, const int32_t *actions_host, uint8_t *mask_host, float *obs_host,
                        int32_t *scalars_host, void *after_stream) {
    return host_step_begin_impl(h, actions_host, mask_host, obs_host, nullptr, scalars_host, after_stream);
}

int jss_host_step_begin_packed(jss_t *h, const int32_t *actions_host, uint8_t *mask_host, uint8_t *wire_host,
                               int32_t *scalars_host, void *after_stream) {
    if (!wire_host || !scalars_host)
        return fail(h, JSS_ERR_INVALID, "jss_host_step_begin_packed: wire_host and scalars_host are required");
    return host_step_begin_impl(h, actions_host, mask_host, nullptr, wire_host, scalars_host, after_stream);
}

int jss_host_step_begin_hybrid(jss_t *h, const int32_t *actions_host, uint8_t *mask_host, uint8_t *wire_host,
                               float *obs_host, int n_dma, int32_t *scalars_host, void *after_stream) {
    if (!wire_host || !obs_host || !scalars_host || n_dma < 0)
        return fail(h, JSS_ERR_INVALID, "jss_host_step_begin_hybrid: wire_host, obs_host, scalars_host and n_dma >= 0 are required");
    return host_step_begin_impl(h, actions_host, mask_host, obs_host, wire_host, scalars_host, after_stream, n_dma);
}

int64_t jss_host_wire_stride(jss_t *h) {
    if (!h || !h->assigned) return JSS_ERR_STATE;
    // 16-byte multiple with >= 6 bytes of slack behind the last record (the host expansion loads 16 bytes per job)
    return round_up(JSS_WIRE_JOB_BYTES * h->p.jobs_max + 6, 16);
}

int jss_host_expand_obs(jss_t *h, const uint8_t *wire_host, const int32_t *scalars_host, float *obs_host) {
    return jss_host_expand_obs_range(h, wire_host, scalars_host, obs_host, 0, h ? h->n_envs : 0);
}

int jss_host_expand_obs_range(jss_t *h, const uint8_t *wire_host, const int32_t *scalars_host, float *obs_host,
                              int env_begin, int env_end) {
    if (!h || !h->assigned) return fail(h, JSS_ERR_STATE, "jss_host_expand_obs: jss_assign must be called first");
    if (!wire_host || !scalars_host || !obs_host || env_begin < 0 || env_end > h->n_envs || env_begin > env_end)
        return fail(h, JSS_ERR_INVALID, "jss_host_expand_obs: bad arguments");
    JssHostExpandArgs a{wire_host, jss_host_wire_stride(h), scalars_host, h->env_inst.data(), h->insts.data(),
                        h->len.data(), obs_host, h->p.jobs_max, env_begin, env_end};
    jss_host_expand_impl(&a);
    return JSS_OK;
}

int jss_host_configure(int threads, int bind_numa_of_device) {
    std::vector<int> cpus;
#ifndef JSS_EMU
    if (bind_numa_of_device >= 0) {
        // CPUs of the NUMA node the GPU hangs off (pinned buffers and the expansion threads stay local to it)
        char bus[32] = {0};
        if (cudaDeviceGetPCIBusId(bus, sizeof bus, bind_numa_of_device) == cudaSuccess) {
            for (char *c = bus; *c; c++) *c = (char)tolower(*c);
            char path[160];
            snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
            int node = -1;
            if (FILE *f = fopen(path, "r")) { if (fscanf(f, "%d", &node) != 1) node = -1; fclose(f); }
            if (node >= 0) {
                snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
                if (FILE *f = fopen(path, "r")) {
                    int a = 0, b = 0;
                    char sep = 0;
                    cpu_set_t allowed;
                    const bool have = sched_getaffinity(0, sizeof allowed, &allowed) == 0;
                    while (fscanf(f, "%d", &a) == 1) {
                        b = a;
                        if (fscanf(f, "%c", &sep) == 1 && sep == '-') { if (fscanf(f, "%d", &b) != 1) b = a; if (fscanf(f, "%c", &sep) != 1) sep = 0; }
                        for (int c = a; c <= b; c++)
                            if (!have || CPU_ISSET(c, &allowed)) cpus.push_back(c);
                        if (sep != ',') break;
                    }
                    fclose(f);
                }
            }
        }
        (void)cudaGetLastError();
    }
#else
    (void)bind_numa_of_device;
#endif
    jss_host_pool_configure(threads, cpus.data(), (int)cpus.size());
    return (int)cpus.size();
}

int jss_host_threads(void) { return jss_host_pool_size(); }

int jss_host_set_simd(int level) { jss_host_simd_cap(level); return JSS_OK; }

int jss_host_wait(jss_t *h, int what) {
    int rc = check_ready(h);
    if (rc) return rc;
    if (!h->pipe_ready) return fail(h, JSS_ERR_STATE, "jss_host_wait: no jss_host_step_begin in flight");
    if (what == JSS_WAIT_MASK) JSS_CUDA(h, cudaEventSynchronize(h->ev_mask));
    else if (what == JSS_WAIT_OBS) JSS_CUDA(h, cudaEventSynchronize(h->ev_obs[h->pipe_cur]));
    else if (what == JSS_WAIT_OBS_PREV) JSS_CUDA(h, cudaEventSynchronize(h->ev_obs[h->pipe_cur ^ 1]));
    else if (what == JSS_WAIT_WIRE) JSS_CUDA(h, cudaEventSynchronize(h->ev_wire));
    else return fail(h, JSS_ERR_INVALID, "jss_host_wait: unknown selector %d", what);
    return JSS_OK;
}

int jss_stats(jss_t *h, int64_t *out_host, void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    if (!out_host) return fail(h, JSS_ERR_INVALID, "jss_stats: out_host is NULL");
    cudaStream_t st = (cudaStream_t)stream;
    unsigned long long init[JSS_STATS_LEN] = {0, 0, 0, ~0ull, 0, 0, 0, 0};
    JSS_CUDA(h, cudaMemcpyAsync(h->d_stats, init, sizeof init, cudaMemcpyHostToDevice, st));
    const int threads = 256;
    const int blocks = std::min((h->n_envs + threads - 1) / threads, h->sm_count * 4);
    JssLaunch a{};                       // every tile of the batch
    a.tile_end = h->n_tiles;
    if (h->p.uniform_inst >= 0) a.uni = h->insts[h->p.uniform_inst];
    JSS_LAUNCH(jss_stats_kernel, blocks, threads, 0, st, h->p, a, h->d_stats);
    JSS_CUDA(h, cudaGetLastError());
    h->launches += 1;
    unsigned long long res[JSS_STATS_LEN];
    JSS_CUDA(h, cudaMemcpyAsync(res, h->d_stats, sizeof res, cudaMemcpyDeviceToHost, st));
    JSS_CUDA(h, cudaStreamSynchronize(st));
    for (int i = 0; i < JSS_STATS_LEN; i++) out_host[i] = (int64_t)res[i];
    if (res[3] == ~0ull) out_host[3] = INT64_MAX;
    return JSS_OK;
}

int jss_export_state(jss_t *h, void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    JssLaunch a{};
    a.mode = JSS_MODE_EXPORT;
    return launch_all(h, a, (cudaStream_t)stream);
}

int jss_import_state(jss_t *h, const uint8_t *env_mask_dev, void *stream) {
    int rc = check_ready(h, stream);
    if (rc) return rc;
    JssLaunch a{};
    a.mode = JSS_MODE_IMPORT;
    a.env_mask = env_mask_dev;
    return launch_all(h, a, (cudaStream_t)stream);
}

int jss_host_masked_random(const uint8_t *mask_host, int n, int width, int64_t row_stride, uint64_t seed,
                           uint64_t env_id_base, uint64_t step_index, int32_t *actions_host) {
    if (!mask_host || !actions_host || n < 0 || width <= 0 || row_stride < width) return JSS_ERR_INVALID;
    jss_host_masked_random_impl(mask_host, n, width, row_stride, seed, env_id_base, step_index, actions_host);   // persistent pool
    return JSS_OK;
}

}  // extern "C"
