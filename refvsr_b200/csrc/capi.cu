// C-ABI glue: error reporting, launch accounting and the rv_conv2d dispatcher.
#include <cstdarg>

#include "common.cuh"

namespace rv {

thread_local std::string g_last_error;
std::atomic<uint64_t> g_launches{0};

int fail(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
  return code;
}

int conv2d_simt(const rv_conv_desc* d, cudaStream_t st);
int conv2d_tc(const rv_conv_desc* d, cudaStream_t st);
int conv2d_tc_plan(const rv_conv_desc* d, int max_smem, int num_sms, int* out);
int conv2d_tc_epi_depth(const rv_conv_desc* d, int max_smem, int num_sms, int* depth);
int conv2d_tc_out_store(const rv_conv_desc* d, int max_smem, int num_sms, int* kind);
int set_conv_cta_cap(int cap);
int set_conv_smem_cap(int bytes);
int set_conv_consumers(int n);
int conv2d_tc_consumers(const rv_conv_desc* d, int max_smem, int num_sms, int* out);

}  // namespace rv

extern "C" const char* rv_last_error(void) { return rv::g_last_error.c_str(); }
extern "C" int rv_version(void) { return 100; }
extern "C" uint64_t rv_launch_count(void) { return rv::g_launches.load(); }

// the batch fields of a descriptor (rv_conv_desc::n and the image strides)
static int check_batch(const rv_conv_desc* d) {
  RV_REQUIRE(d->n >= 0, "rv_conv2d: n=%d must be >= 0", d->n);
  RV_REQUIRE(d->n <= 1 || (d->bs_src0 > 0 && (!d->src1 || d->bs_src1 > 0) && (!d->gate || d->bs_gate > 0) &&
                           (!d->res || d->bs_res > 0) && d->bs_out > 0),
             "rv_conv2d: n=%d needs a positive image stride for every operand", d->n);
  return RV_OK;
}

extern "C" int rv_conv2d(const rv_conv_desc* d, void* stream) {
  RV_REQUIRE(d != nullptr, "rv_conv2d: null descriptor");
  RV_REQUIRE(d->src0 && d->wpack && d->bias && d->out, "rv_conv2d: null src0/wpack/bias/out");
  RV_REQUIRE(d->H > 0 && d->W > 0 && d->c0 > 0 && d->cout > 0 && d->kh > 0 && d->kw > 0 && d->stride > 0,
             "rv_conv2d: bad geometry H=%d W=%d c0=%d cout=%d k=%dx%d stride=%d", d->H, d->W, d->c0,
             d->cout, d->kh, d->kw, d->stride);
  if (const int rc = check_batch(d)) return rc;
  if (d->impl == RV_CONV_IMPL_TC) return rv::conv2d_tc(d, (cudaStream_t)stream);
  RV_REQUIRE(d->ps_order == 0 || d->impl == RV_CONV_IMPL_TC, "rv_conv2d: ps_order=%d is a tensor-core weight order", d->ps_order);
  RV_REQUIRE(d->impl == RV_CONV_IMPL_SIMT, "rv_conv2d: unknown impl %d", d->impl);
  if (d->n <= 1) return rv::conv2d_simt(d, (cudaStream_t)stream);
  // the CUDA-core kernel has no image dimension: one launch per image
  for (int i = 0; i < d->n; ++i) {
    rv_conv_desc e = *d;
    auto at = [i](const void* q, int64_t bs, int esz) {
      return q ? static_cast<const void*>(static_cast<const char*>(q) + (size_t)i * bs * esz) : nullptr;
    };
    const int isz = rv::dtype_size(d->in_dtype);
    e.src0 = at(d->src0, d->bs_src0, isz);
    e.src1 = at(d->src1, d->bs_src1, isz);
    e.gate = at(d->gate, d->bs_gate, isz);
    e.res = at(d->res, d->bs_res, rv::dtype_size(d->res_dtype));
    e.out = const_cast<void*>(at(d->out, d->bs_out, rv::dtype_size(d->out_dtype)));
    e.n = 1;
    if (const int rc = rv::conv2d_simt(&e, (cudaStream_t)stream)) return rc;
  }
  return RV_OK;
}

extern "C" int rv_set_conv_cta_cap(int cap) { return rv::set_conv_cta_cap(cap); }
extern "C" int rv_set_conv_smem_cap(int bytes) { return rv::set_conv_smem_cap(bytes); }
extern "C" int rv_set_conv_consumers(int n) { return rv::set_conv_consumers(n); }

extern "C" int rv_conv2d_tc_plan(const rv_conv_desc* d, int max_smem_optin, int num_sms, int32_t* out8) {
  RV_REQUIRE(d != nullptr && out8 != nullptr && max_smem_optin > 0 && num_sms > 0, "rv_conv2d_tc_plan: bad arguments");
  if (const int rc = check_batch(d)) return rc;
  return rv::conv2d_tc_plan(d, max_smem_optin, num_sms, out8);
}

extern "C" int rv_conv2d_tc_epi_depth(const rv_conv_desc* d, int max_smem_optin, int num_sms, int32_t* depth) {
  RV_REQUIRE(d != nullptr && depth != nullptr && max_smem_optin > 0 && num_sms > 0, "rv_conv2d_tc_epi_depth: bad arguments");
  if (const int rc = check_batch(d)) return rc;
  return rv::conv2d_tc_epi_depth(d, max_smem_optin, num_sms, depth);
}

extern "C" int rv_conv2d_tc_out_store(const rv_conv_desc* d, int max_smem_optin, int num_sms, int32_t* kind) {
  RV_REQUIRE(d != nullptr && kind != nullptr && max_smem_optin > 0 && num_sms > 0, "rv_conv2d_tc_out_store: bad arguments");
  if (const int rc = check_batch(d)) return rc;
  return rv::conv2d_tc_out_store(d, max_smem_optin, num_sms, kind);
}

extern "C" int rv_conv2d_tc_consumers(const rv_conv_desc* d, int max_smem_optin, int num_sms, int32_t* out4) {
  RV_REQUIRE(d != nullptr && out4 != nullptr && max_smem_optin > 0 && num_sms > 0, "rv_conv2d_tc_consumers: bad arguments");
  if (const int rc = check_batch(d)) return rc;
  return rv::conv2d_tc_consumers(d, max_smem_optin, num_sms, out4);
}
