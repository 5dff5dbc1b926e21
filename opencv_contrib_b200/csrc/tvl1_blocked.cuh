// tvl1_blocked.cuh -- temporally blocked Dual TV-L1 inner loop (gamma == 0).
//
// Replaces estimateUKernel + estimateDualVariablesKernel (modules/cudaoptflow/src/cuda/
// tvl1flow.cu:209-348), which the reference launches once per inner iteration (88 B/px of HBM
// traffic per iteration), by one kernel that advances a 64x64 pixel region K iterations per HBM
// pass with the whole primal/dual state held in registers.
//
// Geometry.  One CTA = 512 threads = one 64x64 region = (64-2K)^2 output tile + K-pixel halo.
// Each iteration consumes one halo pixel per side (u_new(x) needs p(x-1), p_new(x) needs
// u_new(x+1)), so after K iterations exactly the centre tile is valid; values there are
// bit-identical to K separate full-image passes because every pixel sees the same operands in the
// same order (tvl1_math.cuh).  Image borders need no halo: the reference's border rules (zero
// ghost for the backward differences, zero forward difference on the last row/column) cut the
// dependency.
//
// Thread mapping.  tid -> (lx = tid & 15, tr = tid >> 4); the thread owns pixels
// x in [4*lx, 4*lx+3], y in {2*tr, 2*tr+1} of the region: 8 pixels x 10 values = 80 registers.
// Neighbours inside the 4x2 micro-tile are registers; x-neighbours come from the adjacent lane
// (__shfl within 16-lane rows); y-neighbours cross warps through a 32 KB shared-memory exchange
// (one float4 row per thread and plane), two __syncthreads per iteration.
#pragma once
#include "common.cuh"
#include "tvl1_math.cuh"

namespace b2f {

struct Tvl1State {
    Plane u1, u2, p11, p12, p21, p22;
};

struct Tvl1BlockedPlanes {
    Plane I1wx, I1wy, grad, rho_c;
    Tvl1State s[2];  // ping-pong: a pass reads s[cur], writes s[cur^1]
};

enum { TVL1_REGION = 64, TVL1_KMAX = 12, TVL1_BLOCK_THREADS = 512 };

// Opt the kernels into >48 KB dynamic shared memory on the current device (once per device).
void tvl1_blocked_init(Ctx &c);
// K fused iterations for the next launch.
int tvl1_blocked_pick_k(int knob, int remaining, int rows, int cols);
// One HBM pass: `iters` iterations from state s[cur] into s[cur^1].
void tvl1_blocked_launch(Ctx &c, int cls, const Tvl1BlockedPlanes &B, int cur, int rows, int cols,
                         const Tvl1Scalars &k, int iters);


// ---- persistent TMA variant ----
// Opaque per-(level, direction) descriptor block (10 input and 6 output CUtensorMaps), built once per workspace.
size_t tvl1_tma_maps_bytes();
bool tvl1_tma_build_maps(void *dst, const Tvl1BlockedPlanes &B, int cur, int rows, int cols);
void tvl1_tma_launch(Ctx &c, int cls, const void *maps, const Tvl1BlockedPlanes &B, int cur, int rows, int cols,
                     const Tvl1Scalars &k, int iters, int num_sms);

// Same kernel, iteration count read from device memory when the pass runs (device-side convergence loop).
void tvl1_tma_launch_dev(Ctx &c, int cls, const void *maps, const Tvl1BlockedPlanes &B, int cur, int rows, int cols,
                         const Tvl1Scalars &k, const int *iters_dev, int num_sms);

}  // namespace b2f
