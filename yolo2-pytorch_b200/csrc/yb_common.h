// Host-side helpers shared by the C-ABI translation units: thread-local error string, argument
// checks, launch checks.  Every exported function returns 0 on success, a cudaError_t (> 0) on a
// CUDA failure or a negative library code; the message is available through yb_last_error().
#pragma once
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>

#define YB_ERR_BAD_ARG (-1)
#define YB_ERR_UNSUPPORTED (-2)
#define YB_ERR_DRIVER (-3)

namespace yb {
char* err_buf();               // thread-local, 512 bytes
int fail(int code, const char* fmt, ...);
int check_launch(const char* what);   // cudaGetLastError() -> code + message
int sm_count();                // cached multiProcessorCount of the current device
int* debug_word_device();      // host-mapped int[4] (device pointer), nullptr if unavailable
// the 1x1 unit a conv launch runs in its epilogue (yb_conv_bn_act_chain_fwd): fp16 weight [cout][Cin2 = the conv's Cout], its
// scale / shift / leaky slope
struct ConvChain {
  const void* w;
  const float* scale;
  const float* shift;
  float slope;
  int cout;
};
}  // namespace yb

#define YB_REQUIRE(cond, ...)                                   \
  do {                                                          \
    if (!(cond)) return yb::fail(YB_ERR_BAD_ARG, __VA_ARGS__);  \
  } while (0)

#define YB_CUDA(expr)                                                                          \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) return yb::fail(static_cast<int>(_e), "%s: %s", #expr, cudaGetErrorString(_e)); \
  } while (0)
