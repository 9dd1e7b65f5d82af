#include "nl_error.h"

#include <cstdio>
#include <cstring>

namespace {
thread_local char g_err[512] = "";
}

int nl_set_error(const char *msg) { return nl_set_error_code(NL_ERR_INVALID, msg); }

int nl_set_error_code(int code, const char *msg) {
    std::snprintf(g_err, sizeof(g_err), "%s", msg ? msg : "");
    return code;
}

extern "C" const char *nl_last_error(void) { return g_err; }
extern "C" int nl_version(void) { return 100; }

#include <cstddef>
extern "C" void nl_abi_sizes(int32_t out[4]) {
    out[0] = (int32_t)sizeof(nl_render_stats);
    out[1] = (int32_t)offsetof(nl_render_stats, n_samples);
    out[2] = (int32_t)sizeof(nl_render_args);
    out[3] = (int32_t)sizeof(nl_mlp_weights);
}

extern "C" void nl_abi_sizes_batch(int32_t out[2]) {
    out[0] = (int32_t)sizeof(nl_batch_args);
    out[1] = NL_BATCH_MAX_PROBLEMS;
}

extern "C" void nl_abi_sizes_score(int32_t out[1]) { out[0] = NL_SCORE_MAX_PROBLEMS; }
