#include "common.cuh"
namespace b200 {
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof(g_err), fmt, ap); va_end(ap);
}
const char* last_error() { return g_err; }
thread_local int64_t* g_launch_counter = nullptr;
}
