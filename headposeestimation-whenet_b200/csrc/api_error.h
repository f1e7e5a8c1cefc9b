// api_error.h - the C ABI's error reporting, shared by every entry-point translation unit (whenet_*, whenet_det_*):
// a failing call stores its message in ONE thread-local buffer that whenet_last_error() returns, and returns its code.
#pragma once
#include <cstdarg>
#include <cstdio>

namespace whenet {
namespace api {

inline thread_local char g_err[512] = "";

inline int fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

}  // namespace api
}  // namespace whenet
