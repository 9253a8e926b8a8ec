// Phase probe of the fused wgmma rollout (rollout_tc2.cuh).  Off unless the library is compiled with
// -DGOPS_TC2_PHASE_PROBE (tools/tc2_phase_probe.py makes such a build of its own); in the default build every call
// below is empty and the kernels are the same machine code as without it.
//
// With the probe on, thread 0 of every warpgroup reads clock64() at the phase boundaries of each horizon step and sums
// the cycles between them per phase.  At the end of the kernel the sums are added over all warpgroups of the launch and
// the last CTA to finish prints one line:
//   tc2probe alg=<alg> wgs=<warpgroups> fwd_steps=<n> rev_steps=<n> <phase>=<cycles> ...
// (steps and cycles summed over the warpgroups; the tool divides).
#pragma once
#ifdef GOPS_TC2_PHASE_PROBE
#include <cstdio>
#endif

namespace gops {
namespace tc2 {

enum Phase {
  kFwdL1,    // forward step: observation planes (fixed-chain kernel: A words in registers), layer 1
  kFwdL2,    // forward step: layer 2 + output layer
  kFwdDyn,   // forward step: action, wrapped model step, tape (owner lanes)
  kRevL1,    // reverse step: observation planes, layer 1 recompute (issue and epilogue)
  kRevAdj,   // reverse step: wrapped model-step adjoint (owner lanes, overlapped with the layer-1 wgmma)
  kRevL2,    // reverse step: layer 2 recompute + output (fixed-chain kernel: A words in registers, stored to the H1
             // planes after the issue), delta2 epilogue, dW3
  kRevD2,    // reverse step: delta2 . W2, dW2 / db2
  kRevD1,    // reverse step: delta1, input gradient, dW1 / db1
  kPhases
};

#ifdef GOPS_TC2_PHASE_PROBE
static __device__ unsigned long long g_probe_cyc[kPhases + 2];
static __device__ unsigned int g_probe_done;

struct Probe {
  bool on;                 // thread 0 of the warpgroup
  long long last;
  unsigned long long cyc[kPhases];
  unsigned fsteps, rsteps;
  __device__ __forceinline__ void init(int t) {
    on = t == 0;
    last = 0;
    fsteps = rsteps = 0;
#pragma unroll
    for (int i = 0; i < kPhases; ++i) cyc[i] = 0;
  }
  __device__ __forceinline__ void mark() {
    if (on) last = clock64();
  }
  __device__ __forceinline__ void stamp(int ph) {
    if (on) {
      const long long now = clock64();
      cyc[ph] += (unsigned long long)(now - last);
      last = now;
    }
  }
  __device__ __forceinline__ void step(bool fwd) {
    if (on) (fwd ? fsteps : rsteps) += 1;
  }
  // all threads of the CTA call it once, at the end of the kernel
  __device__ __forceinline__ void finish(int alg, int wgs) {
    if (on) {
#pragma unroll
      for (int i = 0; i < kPhases; ++i) atomicAdd(&g_probe_cyc[i], cyc[i]);
      atomicAdd(&g_probe_cyc[kPhases], (unsigned long long)fsteps);
      atomicAdd(&g_probe_cyc[kPhases + 1], (unsigned long long)rsteps);
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0 && atomicAdd(&g_probe_done, 1u) == gridDim.x - 1) {
      __threadfence();
      unsigned long long c[kPhases + 2];
#pragma unroll
      for (int i = 0; i < kPhases + 2; ++i) c[i] = atomicExch(&g_probe_cyc[i], 0ull);
      printf("tc2probe alg=%d wgs=%d fwd_steps=%llu rev_steps=%llu fwd_l1=%llu fwd_l2=%llu fwd_dyn=%llu rev_l1=%llu "
             "rev_adj=%llu rev_l2=%llu rev_d2=%llu rev_d1=%llu\n",
             alg, wgs * (int)gridDim.x, c[kPhases], c[kPhases + 1], c[kFwdL1], c[kFwdL2], c[kFwdDyn], c[kRevL1],
             c[kRevAdj], c[kRevL2], c[kRevD2], c[kRevD1]);
      g_probe_done = 0;
    }
  }
};
#else
struct Probe {
  __device__ __forceinline__ void init(int) {}
  __device__ __forceinline__ void mark() {}
  __device__ __forceinline__ void stamp(int) {}
  __device__ __forceinline__ void step(bool) {}
  __device__ __forceinline__ void finish(int, int) {}
};
#endif

}  // namespace tc2
}  // namespace gops
