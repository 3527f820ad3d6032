// errors.h -- the library's one error channel.  Host only, not part of the C ABI.
//
// Every entry point that returns non-zero first writes its reason into uhc_err(), the calling thread's one error text, and every
// uhc_*_last_error() reads it (step_kernel.cu).  A call that fails because a library call it made failed prefixes that call's text
// with what it was doing (uhc_err_prefix).  Clean-up after a failure writes nothing, so the text stays the failure's.
#pragma once
#include <cuda_runtime.h>
#include <string>

// inline: one definition for the whole library, whichever object file (-fmad=false or not) the caller is in
inline std::string &uhc_err() { static thread_local std::string text; return text; }

// a library call failed and wrote its text: "what: <its text>", -1
inline int uhc_err_prefix(const char *what) { uhc_err().insert(0, std::string(what) + ": "); return -1; }

// a CUDA runtime call: on failure "<the call>: <the CUDA error>", -1
#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { uhc_err() = std::string(#x) + ": " + cudaGetErrorString(e_); return -1; } } while (0)
