// config.cpp -- see config.h
#include "config.h"

#include <cstdlib>
#include <cstring>
#include <mutex>

#include "../../include/b200spmv.h"

namespace b200 {

static int parse_csr_kernel(const char* e) {
    if (!e || !e[0] || !strcmp(e, "auto")) return -1;
    if (!strcmp(e, "tile")) return 0;
    if (!strcmp(e, "pipe")) return 1;
    if (!strcmp(e, "ws")) return 2;
    if (!strcmp(e, "rowwise")) return 3;
    if (!strcmp(e, "seg")) return 5;
    return -2;
}
static int parse_coo_kernel(const char* e) {
    if (!e || !e[0] || !strcmp(e, "auto")) return -1;
    if (!strcmp(e, "tile")) return 0;
    if (!strcmp(e, "seg")) return 1;
    return -2;
}
static bool truthy(const char* e) { return e && e[0] && e[0] != '0'; }

static int apply(Config& c, const char* key, const char* value) {
    if (!strcmp(key, "B200SPMV_CSR_KERNEL")) { int v = parse_csr_kernel(value); if (v == -2) return -1; c.csr_kernel = v; return 0; }
    if (!strcmp(key, "B200SPMV_COO_KERNEL")) { int v = parse_coo_kernel(value); if (v == -2) return -1; c.coo_kernel = v; return 0; }
    if (!strcmp(key, "B200SPMV_TILE_ORDER")) { c.tile_scatter = value && !strcmp(value, "scatter"); return 0; }
    if (!strcmp(key, "B200SPMV_PDL")) { c.pdl = truthy(value); return 0; }
    if (!strcmp(key, "B200SPMV_SEG_DENSE")) { c.seg_dense = (value && value[0]) ? atoi(value) : 24; if (c.seg_dense < 1) c.seg_dense = 1; return 0; }
    if (!strcmp(key, "B200SPMV_FLAT")) {
        if (!value || !value[0] || !strcmp(value, "auto")) c.flat = -1;
        else if (!strcmp(value, "on")) c.flat = 1;
        else if (!strcmp(value, "off")) c.flat = 0;
        else return -1;
        return 0;
    }
    if (!strcmp(key, "B200SPMV_SHORT")) {
        if (!value || !value[0] || !strcmp(value, "auto")) c.short_rows = -1;
        else if (!strcmp(value, "on")) c.short_rows = 1;
        else if (!strcmp(value, "off")) c.short_rows = 0;
        else return -1;
        return 0;
    }
    if (!strcmp(key, "B200SPMV_FLAT_QUIET")) { c.flat_quiet_permille = (value && value[0]) ? atoi(value) : 350; return 0; }
    if (!strcmp(key, "B200SPMV_SELL_GENERIC")) { c.sell_generic = truthy(value); return 0; }
    if (!strcmp(key, "B200SPMV_GENERIC")) {
        if (!value || !value[0] || !strcmp(value, "csr") || !strcmp(value, "on") || !strcmp(value, "1")) c.generic = 1;
        else if (!strcmp(value, "off") || !strcmp(value, "0")) c.generic = 0;
        else if (!strcmp(value, "all") || !strcmp(value, "2")) c.generic = 2;
        else return -1;
        return 0;
    }
    if (!strcmp(key, "B200SPMV_ZCSR")) {
        if (!value || !value[0] || !strcmp(value, "auto")) c.zcsr = 0;
        else if (!strcmp(value, "on")) c.zcsr = 1;
        else return -1;
        return 0;
    }
    if (!strcmp(key, "B200SPMV_DENSE")) {
        if (!value || !value[0] || !strcmp(value, "auto")) c.dense = 0;
        else if (!strcmp(value, "on")) c.dense = 1;
        else return -1;
        return 0;
    }
    if (!strcmp(key, "B200SPMV_BANDED")) {
        if (!value || !value[0] || !strcmp(value, "auto")) c.banded = 0;
        else if (!strcmp(value, "on")) c.banded = 1;
        else return -1;
        return 0;
    }
    if (!strcmp(key, "B200SPMV_ILU0")) {
        if (!value || !value[0] || !strcmp(value, "auto")) c.ilu0 = 0;
        else if (!strcmp(value, "on")) c.ilu0 = 1;
        else return -1;
        return 0;
    }
    if (!strcmp(key, "B200SPMV_SPGEMM")) {
        if (!value || !value[0] || !strcmp(value, "auto")) c.spgemm = 0;
        else if (!strcmp(value, "on")) c.spgemm = 1;
        else return -1;
        return 0;
    }
    return -1;
}

Config& config() {
    static Config c;
    static std::once_flag once;
    std::call_once(once, [] {
        static const char* keys[] = {"B200SPMV_CSR_KERNEL", "B200SPMV_COO_KERNEL", "B200SPMV_TILE_ORDER", "B200SPMV_PDL",
                                     "B200SPMV_SEG_DENSE", "B200SPMV_SELL_GENERIC", "B200SPMV_FLAT", "B200SPMV_FLAT_QUIET", "B200SPMV_SHORT", "B200SPMV_GENERIC",
                                     "B200SPMV_ZCSR", "B200SPMV_DENSE", "B200SPMV_BANDED", "B200SPMV_ILU0", "B200SPMV_SPGEMM"};
        for (const char* k : keys)
            if (const char* v = getenv(k)) apply(c, k, v);
    });
    return c;
}

Stats& stats() {
    static Stats s;
    return s;
}

}  // namespace b200

extern "C" {

int b200spmv_set_option(const char* key, const char* value) {
    if (!key) return -1;
    return b200::apply(b200::config(), key, value);
}

void b200spmv_get_stats(uint64_t* native_calls, uint64_t* forwarded_calls, uint64_t* analyze_calls) {
    b200::Stats& s = b200::stats();
    if (native_calls) *native_calls = s.native_calls;
    if (forwarded_calls) *forwarded_calls = s.forwarded_calls;
    if (analyze_calls) *analyze_calls = s.analyze_calls;
}

void b200spmv_reset_stats(void) { b200::stats() = b200::Stats(); }

const char* b200spmv_last_csr_kernel(void) { return b200::stats().last_csr_kernel; }

}  // extern "C"
