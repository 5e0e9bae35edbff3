// Shared by the shims: the entries are extern "C", take raw device pointers, a stream and sizes, and return
// cudaGetLastError() after the launch (the reference's launchers return true unconditionally).
#pragma once
#include "cuda_runtime.h"

#define BSREF extern "C" __attribute__((visibility("default")))

// Element codes used by every entry: 0 fp32, 1 fp16 (the reference's ehalf), 2 bf16 (bhalf).
enum { BSREF_F32 = 0, BSREF_F16 = 1, BSREF_BF16 = 2 };
// Index codes: 0 int32, 1 uint16, 2 uint8.
enum { BSREF_I32 = 0, BSREF_U16 = 1, BSREF_U8 = 2 };

static inline int bsref_sms()
{
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return sms;
}

// The one driver-API call the launchers make (cuMemsetD32Async, to clear atomic accumulators) is defined in ew.cu
// through the runtime's driver entry point, so the library loads without linking libcuda.

static inline int bsref_status()
{
    return (int)cudaGetLastError();
}
