// rl_error.h — the library's one error-message formatter.  Plain C++ with no CUDA include: the host-only units
// (rl_match.cpp, rl_rls.cpp) use it as the CUDA units do, and build with a plain C++ compiler.
#pragma once
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>

// printf-style message, cut at 511 bytes; a long message is never cut in the middle of a UTF-8 sequence
inline std::string rl_format(const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    size_t n = strlen(buf), s = n;
    while (s > 0 && ((unsigned char)buf[s - 1] & 0xC0) == 0x80) s--;
    if (s > 0 && (unsigned char)buf[s - 1] >= 0xC0) {
        const unsigned char lead = (unsigned char)buf[s - 1];
        const size_t need = lead >= 0xF0 ? 4 : lead >= 0xE0 ? 3 : 2;
        if (n - (s - 1) < need) buf[s - 1] = 0;
    }
    return buf;
}
