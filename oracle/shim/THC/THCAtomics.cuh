// ORACLE build shim: stand-in for <THC/THCAtomics.cuh>.  The reference kernels only need atomicAdd on float / double,
// both native on sm_90a.
#pragma once
#include <cuda_runtime.h>
