// C-ABI glue: error text, the execution plan (launch list) and version query.
#include <cstdarg>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "conv_sm90.h"

namespace yb {
namespace {
thread_local char g_err[1024] = "";
}
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace yb

using namespace yb;

struct yb_plan {
  struct Step {
    yb_op_desc desc;
    ConvOp* conv;       // non-null for YB_OP_CONV
    AttentionOp* attn;  // non-null for YB_OP_ATTENTION
  };
  std::vector<Step> steps;
  ~yb_plan() {
    for (auto& s : steps) {
      delete s.conv;
      if (s.attn) attention_op_destroy(s.attn);
    }
  }
};

namespace yb {
int conv_kernel(const yb_op_desc& d) {
  if (d.dtype == YB_F8E4M3) return YB_CONV_KERNEL_E4M3;
  return patch_conv_eligible(d) ? YB_CONV_KERNEL_PATCH : YB_CONV_KERNEL_IM2COL;
}

int conv_config(const yb_op_desc& d, yb_conv_info* info) {
  switch (conv_kernel(d)) {
    case YB_CONV_KERNEL_E4M3: return fp8_conv_config(d, info);
    case YB_CONV_KERNEL_PATCH: return patch_conv_config(d, info);
    default: return im2col_conv_config(d, info);
  }
}

int conv_create(const yb_op_desc& d, ConvOp** out) {
  switch (conv_kernel(d)) {
    case YB_CONV_KERNEL_E4M3: return fp8_conv_create(d, out);
    case YB_CONV_KERNEL_PATCH: return patch_conv_create(d, out);
    default: return im2col_conv_create(d, out);
  }
}
}  // namespace yb

extern "C" const char* yb_last_error(void) { return g_err; }
extern "C" int yb_abi_version(void) { return 2; }

extern "C" int yb_conv_chain_supported(const yb_op_desc* op) {
  if (op == nullptr || op->kind != YB_OP_CONV || op->chain == nullptr) return 0;
  return conv_config(*op, nullptr) == YB_OK ? 1 : 0;
}

extern "C" int yb_conv_config(const yb_op_desc* op, yb_conv_info* info) {
  YB_REQUIRE(op != nullptr && info != nullptr && op->kind == YB_OP_CONV, "conv_config: needs a convolution op and an output struct");
  *info = yb_conv_info();
  return conv_config(*op, info);
}

extern "C" int yb_plan_create(const yb_op_desc* ops, int n_ops, yb_plan** plan_out) {
  YB_REQUIRE(ops && n_ops > 0 && plan_out, "plan_create: null/empty arguments");
  yb_plan* plan = new yb_plan();
  for (int i = 0; i < n_ops; ++i) {
    yb_plan::Step st;
    st.desc = ops[i];
    st.conv = nullptr;
    st.attn = nullptr;
    int rc = YB_OK;
    if (ops[i].in == nullptr || ops[i].out == nullptr) {
      set_error("plan_create: op %d has a null tensor", i);
      rc = YB_ERR_INVALID;
    } else if (ops[i].kind == YB_OP_CONV) {
      if (ops[i].weight == nullptr || ops[i].bias == nullptr) {
        set_error("plan_create: conv op %d without weight/bias", i);
        rc = YB_ERR_INVALID;
      } else {
        rc = conv_create(ops[i], &st.conv);   // validates before any driver call
      }
    } else if (ops[i].kind == YB_OP_ATTENTION) {
      rc = attention_op_create(ops[i], &st.attn);   // validates before any driver call
    } else if (ops[i].kind == YB_OP_DWCONV) {
      rc = dwconv_configure_check(ops[i]);
    } else if (ops[i].kind == YB_OP_SE) {
      rc = se_configure_check(ops[i]);
    } else if (ops[i].kind == YB_OP_AVGPOOL) {
      rc = avgpool_configure_check(ops[i]);
    } else if (ops[i].kind == YB_OP_QUANTIZE) {
      rc = quantize_configure_check(ops[i]);
    } else if (ops[i].kind == YB_OP_SPP_POOL || ops[i].kind == YB_OP_UPSAMPLE2X) {
      rc = validate_pool_or_upsample(ops[i]);
    } else {
      set_error("plan_create: op %d has unknown kind %d", i, ops[i].kind);
      rc = YB_ERR_INVALID;
    }
    if (rc != YB_OK) {
      char inner[900];
      strncpy(inner, g_err, sizeof(inner) - 1);
      inner[sizeof(inner) - 1] = 0;
      set_error("op %d: %s", i, inner);
      delete plan;
      return rc;
    }
    plan->steps.push_back(st);
  }
  *plan_out = plan;
  return YB_OK;
}

extern "C" int yb_plan_run_range(yb_plan* plan, int first, int count, void* stream_) {
  YB_REQUIRE(plan != nullptr, "plan_run: null plan");
  YB_REQUIRE(first >= 0 && count >= 0 && first + count <= static_cast<int>(plan->steps.size()),
             "plan_run: range [%d, %d) outside the %zu ops of the plan", first, first + count, plan->steps.size());
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  for (int i = first; i < first + count; ++i) {
    const yb_plan::Step& st = plan->steps[i];
    int rc;
    switch (st.desc.kind) {
      case YB_OP_CONV:
        rc = st.conv->launch(stream);
        break;
      case YB_OP_ATTENTION:
        rc = attention_op_launch(st.attn, stream);
        break;
      case YB_OP_DWCONV:
        rc = dwconv_launch(st.desc, stream);
        break;
      case YB_OP_SE:
        rc = se_launch(st.desc, stream);
        break;
      case YB_OP_AVGPOOL:
        rc = avgpool_launch(st.desc, stream);
        break;
      case YB_OP_QUANTIZE:
        rc = quantize_launch(st.desc, stream);
        break;
      case YB_OP_SPP_POOL:
        rc = spp_pool_launch(st.desc, stream);
        break;
      default:
        rc = upsample2x_launch(st.desc, stream);
        break;
    }
    if (rc != YB_OK) return rc;
  }
  return YB_OK;
}

extern "C" int yb_plan_run(yb_plan* plan, void* stream) {
  YB_REQUIRE(plan != nullptr, "plan_run: null plan");
  return yb_plan_run_range(plan, 0, static_cast<int>(plan->steps.size()), stream);
}

extern "C" int yb_plan_num_launches(const yb_plan* plan) {
  return plan ? static_cast<int>(plan->steps.size()) : 0;
}

extern "C" int yb_plan_destroy(yb_plan* plan) {
  delete plan;
  return YB_OK;
}
