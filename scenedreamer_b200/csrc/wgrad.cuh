// Jobs of the tensor-core weight-gradient kernel (wgrad.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace rf {

constexpr int kWgMaxJobs = 16;

// One output M-tile: out[row0 + r][0 .. 8*a_chunks) += sum_samples Z[sample][8*z_chunk0 + r] * A[sample][.], r < rows.
// A and Z are tiled bf16 records ([item][chunk][128 rows][8]); a_chunks * 8 = k_in (a multiple of 16, <= 272),
// z_chunks <= 16 chunks of the z_chunks_total chunks of Z's items.  nsplit is filled in by launch_wgrad.
struct WgJob {
    const uint16_t *A;
    const uint16_t *Z;
    float *out;
    int a_chunks;
    int z_chunks_total, z_chunk0, z_chunks;
    int ld_out, row0, rows;
    int nsplit;
};

// dW += over n_items work items (128 samples each); `out` buffers must have been zeroed on the stream.
// d_view = {first, count} in live tiles, read ON THE DEVICE (no host round trip): n_items = count * items_per_live, and the
// items of A start at first * items_per_live (Z holds only these items); d_view null: every item up to cap_items, no offset.
// cap_items (the capacity of one view) only sizes the split of the jobs over the CTAs.
int launch_wgrad(WgJob *jobs, int n_jobs, const int32_t *d_view, int items_per_live, long long cap_items, cudaStream_t st);

}  // namespace rf
