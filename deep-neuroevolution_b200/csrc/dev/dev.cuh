// dev.cuh -- helpers of the DEV library libdne_dev.so (self-tests of the wgmma / TMA plumbing).
// Nothing here is part of the product ABI (include/dne.h); the product library libdne.so does not link it.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#define DNE_OK 0
#define DNE_ERR_ARG -1
#define DNE_ERR_CUDA -2

#define DNE_CHECK_ARG(cond, msg)                                              \
    do {                                                                      \
        if (!(cond)) { fprintf(stderr, "%s: %s\n", __func__, msg); return DNE_ERR_ARG; } \
    } while (0)
#define DNE_CUDA(call)                                                        \
    do {                                                                      \
        cudaError_t e__ = (call);                                             \
        if (e__ != cudaSuccess) { fprintf(stderr, "%s: %s -> %s\n", __func__, #call, cudaGetErrorString(e__)); return DNE_ERR_CUDA; } \
    } while (0)
#define DNE_LAUNCH_CHECK1()                                                   \
    do {                                                                      \
        cudaError_t e__ = cudaGetLastError();                                 \
        if (e__ != cudaSuccess) { fprintf(stderr, "%s: launch -> %s\n", __func__, cudaGetErrorString(e__)); return DNE_ERR_CUDA; } \
    } while (0)
