"""The expected matrix of plan settings: which calls and roles refuse which settings (csrc/plan_settings.h).

A plan can carry ten settings that change what its operator is.  Every call or role in ROWS refuses the settings it lists with
GP_E_STATE and one of two messages:
  form "call":            "<call> is not available on <noun> (<setter>)"
  form "factor" / "term": "<call>: <noun> as a <factor|term> is not available (<setter>)"
Settings are tested in the order of SETTINGS, so the low-rank correction, the one setting that coexists with the others, is
reported before the kernel setting beneath it.  test_plan_settings_host.py compares the compiled table with this one, and
test_gpu_plan_settings.py checks every (row, setting) pair on the device.
"""

GP_E_STATE = 7

# (key, noun, setter) in check order
SETTINGS = [
    ("lowrank", "a plan with a low-rank correction", "gp_plan_set_lowrank"),
    ("tasks", "a plan with task indices", "gp_plan_set_tasks"),
    ("kron", "a Kronecker multitask plan", "gp_plan_set_kron"),
    ("deriv", "a derivative-observation plan", "gp_plan_set_deriv"),
    ("product", "a kernel-product plan", "gp_plan_set_product"),
    ("additive", "an additive plan", "gp_plan_set_additive"),
    ("spectral", "a spectral mixture plan", "gp_plan_set_spectral"),
    ("periodic", "a periodic plan", "gp_plan_set_periodic"),
    ("rq", "a rational quadratic plan", "gp_plan_set_hypers_rq"),
    ("poly", "a polynomial plan", "gp_plan_set_hypers_poly"),
]
KEYS = [s[0] for s in SETTINGS]
NOUN = {k: n for k, n, _ in SETTINGS}
SETTER = {k: s for k, _, s in SETTINGS}

_KERNELS = ("additive", "spectral", "periodic", "rq", "poly")
_ALL_BUT = lambda *skip: tuple(k for k in KEYS if k not in skip)   # noqa: E731

# (row id, name the message reports, form, refused settings), in the order of csrc/plan_settings.h
ROWS = [
    ("set_backend", "gp_plan_set_backend", "call", ("deriv", "product", "additive", "spectral")),
    ("set_hypers_rq", "gp_plan_set_hypers_rq", "call", ("tasks", "kron", "deriv", "product", "additive", "spectral", "periodic")),
    ("set_hypers_poly", "gp_plan_set_hypers_poly", "call", ("tasks", "kron", "deriv", "product", "additive", "spectral", "periodic")),
    ("set_comm", "gp_plan_set_comm with more than one rank", "call", ("product",) + _KERNELS),
    ("set_ski", "gp_plan_set_ski", "call", _ALL_BUT("lowrank")),
    ("ski_input_grad", "gp_ski_input_grad", "call", ("lowrank", "tasks", "kron", "deriv", "product")),
    ("set_tasks", "gp_plan_set_tasks", "call", _ALL_BUT("lowrank", "tasks")),
    ("set_tasks_lowrank", "gp_plan_set_tasks", "call", ("lowrank",)),
    ("set_additive", "gp_plan_set_additive", "call", _ALL_BUT("lowrank", "additive")),
    ("set_spectral", "gp_plan_set_spectral", "call", _ALL_BUT("lowrank", "spectral")),
    ("set_periodic", "gp_plan_set_periodic", "call", _ALL_BUT("lowrank", "periodic")),
    ("set_sum", "gp_plan_set_sum", "call", ("tasks", "kron", "deriv", "product", "additive", "spectral", "periodic")),
    ("set_product", "gp_plan_set_product", "call", _ALL_BUT("product")),
    ("set_kron", "gp_plan_set_kron", "call", _ALL_BUT("kron")),
    ("set_deriv", "gp_plan_set_deriv", "call", _ALL_BUT("deriv")),
    ("set_deriv_kind", "gp_plan_set_deriv_kind", "call", _ALL_BUT("deriv")),
    ("set_lowrank", "gp_plan_set_lowrank", "call", ("tasks", "kron", "deriv", "product")),
    ("kmv_input_grad", "gp_kmv_input_grad", "call", _ALL_BUT("rq", "poly")),
    ("kdense_input_grad", "gp_kdense_input_grad", "call", _ALL_BUT("rq", "poly")),
    ("pivoted_cholesky", "gp_pivoted_cholesky", "call", ("lowrank",)),
    ("precond_build", "gp_precond_build", "call", ("lowrank",)),
    ("ciq_precond_build", "gp_ciq_precond_build", "call", ("lowrank",)),
    ("precond_probes", "gp_precond_probes", "call", ("lowrank",)),
    ("bilinear_grad", "gp_bilinear_grad", "call", ("lowrank",)),
    ("mbcg_precond", "gp_mbcg with a preconditioner", "call", ("lowrank",)),
    ("ciq_sqrt_matmul_precond", "gp_ciq_sqrt_matmul_precond", "call", ("lowrank",)),
    # roles: the settings a plan may not carry when another plan takes it in
    ("kron_data", "gp_plan_set_kron (as the data plan)", "call", ("product",) + _KERNELS),
    ("deriv_data", "gp_plan_set_deriv (as the data plan)", "call", ("product",) + _KERNELS),
    ("deriv_kind_data", "gp_plan_set_deriv_kind (as the data plan)", "call", ("product",) + _KERNELS),
    ("kron_data_refresh", "a Kronecker operator (as the data plan)", "call", ("lowrank", "tasks", "rq", "poly")),
    ("deriv_data_refresh", "a derivative operator (as the data plan)", "call", ("lowrank", "tasks")),
    ("product_factor", "gp_plan_set_product", "factor", ("product",) + _KERNELS),
    ("product_factor_refresh", "kernel product", "factor", ("lowrank", "tasks", "rq", "poly")),
    ("sum_term", "gp_plan_set_sum", "term", ("product", "additive", "spectral")),
    ("sum_term_refresh", "kernel sum", "term", ("tasks",)),
]
ROW = {r[0]: r for r in ROWS}


def message(row: str, setting: str) -> str:
    """The message of a refused (row, setting) pair."""
    _, name, form, _ = ROW[row]
    if form == "call":
        return f"{name} is not available on {NOUN[setting]} ({SETTER[setting]})"
    return f"{name}: {NOUN[setting]} as a {form} is not available ({SETTER[setting]})"


def refused(row: str, settings) -> str | None:
    """The setting a row reports for a plan carrying `settings`, or None: the first refused one in check order."""
    mask = ROW[row][3]
    return next((k for k in KEYS if k in settings and k in mask), None)


# Messages the table reworded into its two forms: the text the parent commit of the table printed for the same refusal.
REWORDED = {
    ("set_tasks_lowrank", "lowrank"): "task indices are not available on a plan with a low-rank correction",
    ("kron_data_refresh", "tasks"): "Kronecker plan: a data plan with task indices is not available",
    ("kron_data_refresh", "lowrank"): "Kronecker plan: a data plan with a low-rank correction is not available",
    ("deriv_data_refresh", "tasks"): "derivative plan: a data plan with task indices is not available",
    ("deriv_data_refresh", "lowrank"): "derivative plan: a data plan with a low-rank correction is not available",
    ("product_factor", "product"): "kernel product: a factor that is itself a kernel product is not available",
    ("product_factor_refresh", "tasks"): "kernel product: a factor with task indices is not available",
    ("product_factor_refresh", "lowrank"): "kernel product: a factor with a low-rank correction is not available",
    ("product_factor_refresh", "rq"): "kernel product: a rational quadratic factor is not available (gp_plan_set_hypers_rq)",
    ("product_factor_refresh", "poly"): "kernel product: a polynomial factor is not available (gp_plan_set_hypers_poly)",
    ("sum_term", "product"): "gp_plan_set_sum: a kernel product as a term is not available (gp_plan_set_product)",
    ("sum_term_refresh", "tasks"): "kernel sum: a term with task indices is not available",
}
