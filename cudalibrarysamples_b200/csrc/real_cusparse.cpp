// real_cusparse.cpp -- see real_cusparse.h
#include "real_cusparse.h"

#include <dlfcn.h>

#include <cstdio>
#include <cstdlib>

namespace b200 {

void* open_real_cusparse(const char* tag) {
    const char* path = getenv("B200SPMV_CUSPARSE");
    const char* cands[] = {path, "libcusparse.so.12", "/usr/local/cuda/lib64/libcusparse.so.12", "libcusparse.so"};
    for (const char* c : cands) {
        if (!c || !c[0]) continue;
        if (void* h = dlopen(c, RTLD_NOW | RTLD_LOCAL)) return h;
    }
    fprintf(stderr, "[%s] FATAL: cannot dlopen the real libcusparse.so.12 (%s); set B200SPMV_CUSPARSE\n", tag, dlerror());
    abort();
}

void* real_symbol(void* h, const char* name, const char* tag) {
    void* f = dlsym(h, name);
    if (!f) {
        fprintf(stderr, "[%s] FATAL: real libcusparse lacks %s\n", tag, name);
        abort();
    }
    return f;
}

bool env_flag(const char* name) {
    const char* v = getenv(name);
    return v && v[0] && v[0] != '0';
}

}  // namespace b200
