// bm2_common.cuh — shared declarations of the H100 seed-and-extend library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <string>
#include "bm2_b200.h"

#define BM2_CUDA_OK(expr)                                                                       \
    do {                                                                                        \
        cudaError_t _e = (expr);                                                                \
        if (_e != cudaSuccess) {                                                                \
            bm2_set_error(ctx_for_error, std::string(#expr) + ": " + cudaGetErrorString(_e));   \
            return 1;                                                                           \
        }                                                                                       \
    } while (0)

struct bm2_ctx;
void bm2_set_error(bm2_ctx *ctx, const std::string &msg);

#include "bsw_types.h"

// Sort-and-launch of the thread-per-job BSW kernel over `n` jobs (device arrays).
// perm/keys are scratch of n elements each; cells (device, may be null) accumulates DP cells.
int bsw_launch(bm2_ctx *ctx_for_error, cudaStream_t stream, const BswJob *d_jobs, BswOut *d_out, int n,
               const uint8_t *d_tbase, const uint8_t *d_qbase, const BswParams &prm,
               unsigned long long *d_cells);
size_t bsw_scratch_bytes(int n);
