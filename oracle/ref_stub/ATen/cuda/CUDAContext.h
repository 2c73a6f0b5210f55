// Stub standing in for <ATen/cuda/CUDAContext.h> when the reference's .cu files
// are compiled (unmodified, where they lie in the reference checkout) into
// oracle/_ref/libexllama_ref.so WITHOUT torch.  The reference .cu files only
// need cuBLAS types and the TORCH_CHECK macro from that header.
// TEST INFRASTRUCTURE ONLY (see oracle/Makefile).
#pragma once
#include <cublas_v2.h>
#include <cstdio>
#include <stdexcept>
#ifndef TORCH_CHECK
#define TORCH_CHECK(cond, ...) \
    do { if (!(cond)) { fprintf(stderr, "TORCH_CHECK failed: %s\n", #cond); throw std::runtime_error(#cond); } } while (0)
#endif
