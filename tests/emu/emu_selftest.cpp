// emu_selftest.cpp -- TEST-ONLY kernel with deliberate shared-memory hazards, compiled into the emulation library
// alone.  tests/test_emu_schedules.py runs it to show that jss_emu_set_schedule() changes what such a kernel sees, so
// that the kernels' suites passing under the other schedules means something.
#include "cuda_shim.h"

namespace {
constexpr int kWarps = 8, kPairs = 16;
constexpr int kOut = kWarps * kPairs + kWarps / 2 + 1;   // per block: lane pairs, warp pairs, one unwritten word

// distinct per block, so that a block never mistakes what an earlier one left behind for its own write, and never a
// repeated byte, so that it is never a poison pattern
int marker(int a, int b) { return 0x31000000 + ((int)blockIdx.x << 16) + (a << 8) + b; }

// Per block, with no barrier between a write and its read:
//   lane l < 16 of every warp writes a word that lane 31 - l of the same warp reads;
//   lane 0 of warp w < 4 writes a word that lane 0 of warp 7 - w reads;
//   thread 0 reads a word nothing in this block has written, then writes it.
// out[b * kOut + k] is 1 where the read saw the write, 0 where it did not; the last word is the unwritten one.
__global__ void hazard_kernel(int *out, int) {
    JSS_SMEM_DECL(smem);
    int *lanes = reinterpret_cast<int *>(smem), *warps = lanes + kWarps * kPairs, *unwritten = warps + kWarps / 2;
    int *o = out + blockIdx.x * kOut;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) o[kOut - 1] = *unwritten;
    if (lane < kPairs) lanes[warp * kPairs + lane] = marker(warp, lane);
    if (lane == 0 && warp < kWarps / 2) warps[warp] = marker(kWarps + warp, 0);
    if (lane >= 32 - kPairs) {
        const int writer = 31 - lane;
        o[warp * kPairs + writer] = lanes[warp * kPairs + writer] == marker(warp, writer);
    }
    if (lane == 0 && warp >= kWarps / 2) {
        const int writer = kWarps - 1 - warp;
        o[kWarps * kPairs + writer] = warps[writer] == marker(kWarps + writer, 0);
    }
    __syncthreads();
    if (threadIdx.x == 0) *unwritten = 0x7e57;
}
}  // namespace

// The number of words hazard_kernel writes per block.
extern "C" int jss_emu_selftest_width() { return kOut; }

// Runs `blocks` blocks of hazard_kernel into out[blocks * jss_emu_selftest_width()] and stores in *fresh the first
// word of a new cudaMalloc allocation.  1 <= blocks <= 207.  Returns 0, or -1 if
// `blocks` is out of range or an allocation failed.
extern "C" int jss_emu_selftest(int blocks, int *out, int *fresh) {
    if (blocks < 1 || blocks > 0xcf) return -1;
    int *d_out = nullptr, *d_fresh = nullptr;
    if (cudaMalloc((void **)&d_fresh, sizeof(int)) || cudaMalloc((void **)&d_out, sizeof(int) * kOut * blocks)) return -1;
    cudaMemcpy(fresh, d_fresh, sizeof(int), cudaMemcpyDeviceToHost);
    cudaMemset(d_out, 0xff, sizeof(int) * kOut * blocks);
    JSS_LAUNCH(hazard_kernel, blocks, kWarps * 32, sizeof(int) * kOut, nullptr, d_out, 0);
    cudaMemcpy(out, d_out, sizeof(int) * kOut * blocks, cudaMemcpyDeviceToHost);
    cudaFree(d_out);
    cudaFree(d_fresh);
    return 0;
}
