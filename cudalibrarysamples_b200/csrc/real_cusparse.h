// real_cusparse.h -- how both shims (libb200spmv.so, libb200spsv.so) reach the closed libcusparse.so.12 and read their
// run-time switches.  Compiled into each library with hidden visibility: neither exports it, and neither library needs
// the other to load.
#pragma once

namespace b200 {

// dlopen()s the real library: $B200SPMV_CUSPARSE first, then the usual sonames.  Aborts with a message tagged `tag`
// (e.g. "b200spmv") when none loads: a shim without the real library cannot even create a handle.
__attribute__((visibility("hidden"))) void* open_real_cusparse(const char* tag);

// dlsym()s `name` from the handle open_real_cusparse returned.  Aborts with a message tagged `tag` when the real library
// lacks it: every symbol a shim loads is one it forwards to.
__attribute__((visibility("hidden"))) void* real_symbol(void* h, const char* name, const char* tag);

// true when the environment variable is set to anything but "" or a leading '0' (B200SPMV_FORWARD, B200SPMV_LOG)
__attribute__((visibility("hidden"))) bool env_flag(const char* name);

}  // namespace b200
