// check.h — how the host library fails: it throws.  A caller's bad argument is std::invalid_argument, an invariant nothing
// should reach is std::logic_error, and a CUDA or NCCL call that fails is a DeviceError.  The C API (capi.cc) turns each
// into a status and the message of cnb_last_error(); nothing in the library ends the process.  Destructors free with
// unchecked calls and never throw.  After a DeviceError in the middle of a step the net's state is undefined.
#pragma once
#include <cuda_runtime.h>

#include <cstring>
#include <stdexcept>
#include <string>

namespace cnbhost {

struct DeviceError : std::runtime_error {
  using std::runtime_error::runtime_error;
};

// "<source file>(<line>): <api> error: <expr>: <the library's message>"
[[noreturn]] inline void ThrowDeviceError(const char* file, int line, const char* api, const char* expr, const char* what) {
  const char* slash = strrchr(file, '/');
  throw DeviceError(std::string(slash ? slash + 1 : file) + "(" + std::to_string(line) + "): " + api + " error: " + expr +
                    ": " + what);
}

// ncclGetErrorString of the NCCL the library loaded (convnet.cc)
const char* NcclErrorString(int result);

}  // namespace cnbhost

#define CUDA_CHECK(expr)                                                                                 \
  do {                                                                                                   \
    const cudaError_t _e = (expr);                                                                       \
    if (_e != cudaSuccess) ::cnbhost::ThrowDeviceError(__FILE__, __LINE__, "CUDA", #expr, cudaGetErrorString(_e)); \
  } while (0)

#define NCCL_CHECK(expr)                                                                                 \
  do {                                                                                                   \
    const int _r = (int)(expr);                                                                          \
    if (_r != 0) ::cnbhost::ThrowDeviceError(__FILE__, __LINE__, "NCCL", #expr, ::cnbhost::NcclErrorString(_r)); \
  } while (0)
