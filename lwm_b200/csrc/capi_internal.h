// Internal helpers shared by the C-ABI entry points (status codes, last-error string, device check).
#pragma once
#include <cuda_runtime.h>
#include <type_traits>

enum {
  LWM_OK = 0,
  LWM_ERR_DEVICE = 1,  // not an sm_90 device / no CUDA device: there is no fallback path
  LWM_ERR_SHAPE = 2,
  LWM_ERR_ARG = 3,
  LWM_ERR_CUDA = 4,
};

int lwm_fail(int code, const char* msg);          // records msg, returns code
bool lwm_check_device();                          // true iff current device is compute capability 9.x
int lwm_check_launch(const char* what);           // cudaGetLastError -> status

// with_flags(f, b0, b1, ...) = f(std::bool_constant<b0>{}, std::bool_constant<b1>{}, ...): turns an entry point's
// run-time options into the template arguments of the kernel instance that serves them, in one place.
template <typename F>
static int with_flags(F&& f) {
  return f();
}
template <typename F, typename... Bs>
static int with_flags(F&& f, bool b, Bs... rest) {
  if (b) return with_flags([&](auto... t) { return f(std::true_type{}, t...); }, rest...);
  return with_flags([&](auto... t) { return f(std::false_type{}, t...); }, rest...);
}

// SM count of the H100 SXM: cap of the grid-stride launches (one or a few waves of resident blocks)
constexpr long long kNumSMs = 132;

// attn_decode.cu: fold n_part partials per row ([rows][n_part][128] numerators, [rows][n_part][2] (max_log2, den))
// into one partial per row. Also merges the key splits of attn_fwd.cu's inference mode.
void lwm_decode_merge_partials(const float* o_parts, const float* ml_parts, int n_part, float* o_merged,
                               float* ml_merged, long long rows, cudaStream_t st);
