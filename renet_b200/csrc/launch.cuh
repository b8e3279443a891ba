// Kernel launches with programmatic dependent launch (PDL) and the host-side guard of its hazard rule (DESIGN §4).
//
// A launch with programmatic stream serialisation may start as soon as every CTA of the previous kernel in the stream has
// executed griddepcontrol.launch_dependents (or exited); what it does before its own griddepcontrol.wait then overlaps that
// kernel's tail.  The library's PDL kernels keep three rules:
//   1. trigger after wait: griddepcontrol.launch_dependents only after the kernel's own griddepcontrol.wait, and every CTA
//      executes the wait before it exits.  So when kernel i starts, kernel i - 2 and everything before it have completed;
//   2. pre-wait reads: kernel i reads before its wait only buffers that kernel i - 1 does not write;
//   3. a kernel from outside the library never triggers early (it triggers implicitly at completion), so a foreign kernel,
//      copy or event between two library launches leaves nothing to check.
// Rule 2 is checked here, on the host: per (device, stream) the byte ranges the last early-triggering library launch
// writes are kept, and a launch asks for the attribute only when its pre-wait ranges are disjoint from them.  A stale
// record (foreign work in between) can only turn the attribute off, never on.
#pragma once
#include <initializer_list>
#include <utility>

#include "common.cuh"

namespace renet {

// device bytes [p, p + bytes)
struct DevSpan {
  const void* p;
  int64_t bytes;
};

// RENET_PDL=0 turns programmatic dependent launch off; read per launch, so one process can compare both modes
bool pdl_allowed();
// true when PDL is allowed and no span of `pre_wait` overlaps what the last early-triggering launch on this stream writes
bool pdl_disjoint(cudaStream_t stream, std::initializer_list<DevSpan> pre_wait);
// this launch triggers early and writes `writes`: it becomes the stream's record
void pdl_record(cudaStream_t stream, std::initializer_list<DevSpan> writes);
void count_pdl_launch();

// Launches `kernel`, which keeps rules 1 and 2 for `pre_wait` (what it reads before its griddepcontrol.wait) and writes
// only within `writes`, with the PDL attribute when pdl_disjoint allows it; either way it becomes the stream's record.
template <typename... P, typename... A>
int launch_pdl(const char* name, std::initializer_list<DevSpan> pre_wait, std::initializer_list<DevSpan> writes,
               void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, A&&... args) {
  const bool pdl = pdl_disjoint(stream, pre_wait);
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr.val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cfg.attrs = &attr;
  cfg.numAttrs = pdl ? 1 : 0;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, std::forward<A>(args)...);
  if (e != cudaSuccess) {
    cudaGetLastError();
    set_error("launch of %s failed: %s", name, cudaGetErrorString(e));
    return RENET_ERR_CUDA;
  }
  pdl_record(stream, writes);
  count_launch();
  if (pdl) count_pdl_launch();
  return RENET_OK;
}

// The device side of rule 1
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

}  // namespace renet
