// api_error.h - the C ABI's error reporting, shared by every entry-point translation unit (whenet_*, whenet_det_*):
// a failing call stores its message in ONE thread-local buffer that whenet_last_error() returns, and returns its code.
// Also the argument checks that more than one unit makes.
#pragma once
#include <cstdarg>
#include <cstdio>

#include "../../include/whenet_b200.h"

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

// the yuv_layout argument of the *_yuv_u8 entry points
inline int check_yuv_layout(int yuv_layout) {
    if (yuv_layout != WHENET_YUV_NV12 && yuv_layout != WHENET_YUV_I420)
        return fail(WHENET_EINVAL, "yuv_layout=%d: WHENET_YUV_NV12 (%d) or WHENET_YUV_I420 (%d)", yuv_layout, WHENET_YUV_NV12, WHENET_YUV_I420);
    return 0;
}

// the yuv422_layout argument of the *_yuv422_u8 entry points
inline int check_yuv422_layout(int yuv422_layout) {
    if (yuv422_layout != WHENET_YUV_YUYV && yuv422_layout != WHENET_YUV_UYVY)
        return fail(WHENET_EINVAL, "yuv422_layout=%d: WHENET_YUV_YUYV (%d) or WHENET_YUV_UYVY (%d)", yuv422_layout, WHENET_YUV_YUYV,
                    WHENET_YUV_UYVY);
    return 0;
}

}  // namespace api
}  // namespace whenet
