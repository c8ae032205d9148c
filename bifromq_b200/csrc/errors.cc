// errors.cc — the thread-local error text behind bfq_last_error(), set by every failing call of the C-ABI.
#include <string>

#include "../../include/bfq_gpumatch.h"
#include "codec.h"

namespace bfq {
thread_local std::string g_last_error;
int32_t set_error(int32_t code, const std::string& msg) {
    g_last_error = msg;
    return code;
}
}  // namespace bfq

extern "C" const char* bfq_last_error(void) { return bfq::g_last_error.c_str(); }
