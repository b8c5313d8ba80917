// jss_host.h -- internal interface between jss_api.cu (C-ABI, CUDA) and jss_host.cpp (host helpers, plain C++).
#pragma once
#include <stdint.h>

#include "jss_types.h"

#define JSS_WIRE_JOB_BYTES 10   // packed observation record of one job (layout: jss_host.cpp / env_pack in jss_device.cuh)

struct JssHostExpandArgs {
    const uint8_t *wire;        // [N][wire_stride] packed rows
    int64_t wire_stride;
    const int32_t *scalars;     // [N][4] scalar records (current_time_step at index 2)
    const int32_t *env_inst;    // [N]
    const JssInst *insts;       // the records jss_load_instances filled
    const int32_t *len_pool;    // jobs_length of instance k at insts[k].len_off
    float *obs;                 // [N][jobs_max][7]
    int jobs_max;
    int64_t env_begin, env_end;
};

int jss_host_pool_configure(int threads, const int *cpus, int n_cpus);
int jss_host_pool_size(void);
void jss_host_simd_cap(int level);   // 0 scalar, 1 AVX2, 2 AVX-512 (tests)
void jss_host_parallel_for(int64_t n, int64_t grain, void (*fn)(int64_t, int64_t, void *), void *ctx);
void jss_host_masked_random_impl(const uint8_t *mask_host, int n, int width, int64_t row_stride, uint64_t seed,
                                 uint64_t env_id_base, uint64_t step_index, int32_t *actions_host);
void jss_host_expand_impl(const JssHostExpandArgs *a);
