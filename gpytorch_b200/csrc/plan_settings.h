// plan_settings.h -- the settings that change what a plan's operator is, and which of them every call and role refuses.
// refuse_settings (api.cu) is the one check: it returns GP_E_STATE for the first refused setting in the order of PlanSetting, with
//   "<call> is not available on <noun> (<setter>)"                  (rows without `as`)
//   "<call>: <noun> as a <factor|term> is not available (<setter>)"  (the plan taken in by gp_plan_set_product / gp_plan_set_sum)
// plan_settings (api.cu) is the only code that maps a plan's fields to these bits.  Host code only: includes nothing but stdint.h.
#pragma once
#include <stdint.h>

namespace gp {

// One bit per setting, in check order.  The low-rank correction comes first: it is the one setting that coexists with others (plain,
// RQ, polynomial, periodic, spectral, additive, SKI and sum plans), and a row that refuses both reports it before the kernel setting
// beneath it.
enum PlanSetting : uint32_t {
  PS_LOWRANK = 1u << 0,    // lr_U
  PS_TASKS = 1u << 1,      // tasks
  PS_KRON = 1u << 2,       // kron
  PS_DERIV = 1u << 3,      // deriv
  PS_PRODUCT = 1u << 4,    // backend_req == GP_BACKEND_PRODUCT
  PS_ADDITIVE = 1u << 5,   // add_M
  PS_SPECTRAL = 1u << 6,   // sm_Q
  PS_PERIODIC = 1u << 7,   // per_n
  PS_RQ = 1u << 8,         // kind == GP_RQ
  PS_POLY = 1u << 9,       // kind == GP_POLY
};
constexpr int PS_COUNT = 10;
constexpr uint32_t PS_KERNELS = PS_ADDITIVE | PS_SPECTRAL | PS_PERIODIC | PS_RQ | PS_POLY;
constexpr uint32_t PS_ALL = (1u << PS_COUNT) - 1;

struct SettingName {
  const char* noun;     // what the messages call a plan carrying the setting
  const char* setter;   // the call that gives it
};
constexpr SettingName SETTING_NAMES[PS_COUNT] = {
    {"a plan with a low-rank correction", "gp_plan_set_lowrank"},
    {"a plan with task indices", "gp_plan_set_tasks"},
    {"a Kronecker multitask plan", "gp_plan_set_kron"},
    {"a derivative-observation plan", "gp_plan_set_deriv"},
    {"a kernel-product plan", "gp_plan_set_product"},
    {"an additive plan", "gp_plan_set_additive"},
    {"a spectral mixture plan", "gp_plan_set_spectral"},
    {"a periodic plan", "gp_plan_set_periodic"},
    {"a rational quadratic plan", "gp_plan_set_hypers_rq"},
    {"a polynomial plan", "gp_plan_set_hypers_poly"},
};

// Every call or role that refuses settings; CALL_ROWS[id] is its row (CALL_SET_TASKS_LOWRANK: gp_plan_set_tasks after its SKI and
// kernel-sum checks).
enum CallId {
  CALL_SET_BACKEND, CALL_SET_HYPERS_RQ, CALL_SET_HYPERS_POLY, CALL_SET_COMM_SHARDED, CALL_SET_SKI, CALL_SKI_INPUT_GRAD,
  CALL_SET_TASKS, CALL_SET_TASKS_LOWRANK, CALL_SET_ADDITIVE, CALL_SET_SPECTRAL, CALL_SET_PERIODIC, CALL_SET_SUM,
  CALL_SET_PRODUCT, CALL_SET_KRON, CALL_SET_DERIV, CALL_SET_DERIV_KIND, CALL_SET_LOWRANK, CALL_KMV_INPUT_GRAD,
  CALL_KDENSE_INPUT_GRAD, CALL_PIVOTED_CHOLESKY, CALL_PRECOND_BUILD, CALL_CIQ_PRECOND_BUILD, CALL_PRECOND_PROBES,
  CALL_BILINEAR_GRAD, CALL_MBCG_PRECOND, CALL_CIQ_SQRT_MATMUL_PRECOND,
  // roles: the plan another plan takes in, at set time and when the taking plan re-checks it before a call
  CALL_KRON_DATA, CALL_DERIV_DATA, CALL_DERIV_KIND_DATA, CALL_KRON_DATA_REFRESH, CALL_DERIV_DATA_REFRESH, CALL_PRODUCT_FACTOR,
  CALL_PRODUCT_FACTOR_REFRESH, CALL_SUM_TERM, CALL_SUM_TERM_REFRESH, CALL_COUNT
};

struct CallRow {
  const char* name;    // the call the message names
  const char* as;      // nullptr, or "factor" / "term": the second message form
  uint32_t refuses;    // PlanSetting bits
};
constexpr CallRow CALL_ROWS[CALL_COUNT] = {
    {"gp_plan_set_backend", nullptr, PS_DERIV | PS_PRODUCT | PS_ADDITIVE | PS_SPECTRAL},
    {"gp_plan_set_hypers_rq", nullptr, PS_TASKS | PS_KRON | PS_DERIV | PS_PRODUCT | PS_ADDITIVE | PS_SPECTRAL | PS_PERIODIC},
    {"gp_plan_set_hypers_poly", nullptr, PS_TASKS | PS_KRON | PS_DERIV | PS_PRODUCT | PS_ADDITIVE | PS_SPECTRAL | PS_PERIODIC},
    {"gp_plan_set_comm with more than one rank", nullptr, PS_PRODUCT | PS_KERNELS},
    {"gp_plan_set_ski", nullptr, PS_ALL & ~PS_LOWRANK},
    {"gp_ski_input_grad", nullptr, PS_LOWRANK | PS_TASKS | PS_KRON | PS_DERIV | PS_PRODUCT},
    {"gp_plan_set_tasks", nullptr, PS_ALL & ~(PS_LOWRANK | PS_TASKS)},
    {"gp_plan_set_tasks", nullptr, PS_LOWRANK},
    {"gp_plan_set_additive", nullptr, PS_ALL & ~(PS_LOWRANK | PS_ADDITIVE)},
    {"gp_plan_set_spectral", nullptr, PS_ALL & ~(PS_LOWRANK | PS_SPECTRAL)},
    {"gp_plan_set_periodic", nullptr, PS_ALL & ~(PS_LOWRANK | PS_PERIODIC)},
    {"gp_plan_set_sum", nullptr, PS_TASKS | PS_KRON | PS_DERIV | PS_PRODUCT | PS_ADDITIVE | PS_SPECTRAL | PS_PERIODIC},
    {"gp_plan_set_product", nullptr, PS_ALL & ~PS_PRODUCT},
    {"gp_plan_set_kron", nullptr, PS_ALL & ~PS_KRON},
    {"gp_plan_set_deriv", nullptr, PS_ALL & ~PS_DERIV},
    {"gp_plan_set_deriv_kind", nullptr, PS_ALL & ~PS_DERIV},
    {"gp_plan_set_lowrank", nullptr, PS_TASKS | PS_KRON | PS_DERIV | PS_PRODUCT},
    {"gp_kmv_input_grad", nullptr, PS_ALL & ~(PS_RQ | PS_POLY)},
    {"gp_kdense_input_grad", nullptr, PS_ALL & ~(PS_RQ | PS_POLY)},
    {"gp_pivoted_cholesky", nullptr, PS_LOWRANK},
    {"gp_precond_build", nullptr, PS_LOWRANK},
    {"gp_ciq_precond_build", nullptr, PS_LOWRANK},
    {"gp_precond_probes", nullptr, PS_LOWRANK},
    {"gp_bilinear_grad", nullptr, PS_LOWRANK},
    {"gp_mbcg with a preconditioner", nullptr, PS_LOWRANK},
    {"gp_ciq_sqrt_matmul_precond", nullptr, PS_LOWRANK},
    {"gp_plan_set_kron (as the data plan)", nullptr, PS_PRODUCT | PS_KERNELS},
    {"gp_plan_set_deriv (as the data plan)", nullptr, PS_PRODUCT | PS_KERNELS},
    {"gp_plan_set_deriv_kind (as the data plan)", nullptr, PS_PRODUCT | PS_KERNELS},
    {"a Kronecker operator (as the data plan)", nullptr, PS_LOWRANK | PS_TASKS | PS_RQ | PS_POLY},
    {"a derivative operator (as the data plan)", nullptr, PS_LOWRANK | PS_TASKS},
    {"gp_plan_set_product", "factor", PS_PRODUCT | PS_KERNELS},
    {"kernel product", "factor", PS_LOWRANK | PS_TASKS | PS_RQ | PS_POLY},
    {"gp_plan_set_sum", "term", PS_PRODUCT | PS_ADDITIVE | PS_SPECTRAL},
    {"kernel sum", "term", PS_TASKS},
};

}  // namespace gp
