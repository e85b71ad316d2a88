// Error reporting of the C ABI (include/lookonce_b200.h): an entry point returns 0 or an error code, and
// l2h_last_error() returns the message of the last failure on the calling thread.
#pragma once
#include <cuda_runtime.h>

#include <string>

namespace l2h {

extern thread_local std::string g_err;        // defined in sep_engine.cu
int fail(int code, const std::string& msg);   // records `msg` and returns `code`

}  // namespace l2h

// return error 3 from the enclosing function when a CUDA runtime call fails
#define CK(expr)                                                                                   \
    do {                                                                                           \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess)                                                                     \
            return ::l2h::fail(3, std::string(#expr) + ": " + cudaGetErrorString(_e));             \
    } while (0)
