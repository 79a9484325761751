// l3dpp_wrap.h — what the C wrappers of the host files share (include/l3dpp_capi.h; line3d_sfm.cc, line3d_bin.cc): the copy of a
// message into a caller's buffer.  Host only, header only.
#ifndef L3DPP_WRAP_H_
#define L3DPP_WRAP_H_
#include <cstring>
#include <string>

// s into buf[cap], NUL-terminated and cut to fit; nothing for a null buffer or cap <= 0
inline void l3dpp_copy_str(const std::string& s, char* buf, int cap)
{
    if (buf && cap > 0) { std::strncpy(buf, s.c_str(), cap - 1); buf[cap - 1] = 0; }
}

#endif
