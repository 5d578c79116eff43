"""The table of plan settings (csrc/plan_settings.h) compiled by a host-only program equals plan_settings_oracle.py, and it is the
only place the refusals are written down."""
import os
import re
import shutil
import subprocess

import pytest

import plan_settings_oracle as ps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gpytorch_b200", "csrc")

_PRINT = r"""
#include <stdio.h>
#include "plan_settings.h"
int main() {
  for (int s = 0; s < gp::PS_COUNT; ++s) printf("S|%s|%s\n", gp::SETTING_NAMES[s].noun, gp::SETTING_NAMES[s].setter);
  for (int c = 0; c < gp::CALL_COUNT; ++c) {
    const gp::CallRow& r = gp::CALL_ROWS[c];
    printf("R|%s|%s|", r.name, r.as ? r.as : "call");
    for (int s = 0; s < gp::PS_COUNT; ++s)
      if (r.refuses >> s & 1) printf("%d,", s);
    printf("\n");
  }
  return 0;
}
"""


def _compiler():
    for c in (os.environ.get("CXX"), shutil.which("g++"), shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    return None


def test_compiled_table_equals_the_oracle(tmp_path):
    cc = _compiler()
    if not cc:
        pytest.skip("no host compiler")
    src, exe = tmp_path / "print_table.cpp", tmp_path / "print_table"
    src.write_text(_PRINT)
    r = subprocess.run([cc, "-std=c++17", "-I", CSRC, str(src), "-o", str(exe)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    lines = subprocess.run([str(exe)], capture_output=True, text=True, check=True, timeout=60).stdout.splitlines()
    settings = [tuple(ln.split("|")[1:]) for ln in lines if ln.startswith("S|")]
    assert settings == [(noun, setter) for _, noun, setter in ps.SETTINGS]
    rows = []
    for ln in lines:
        if ln.startswith("R|"):
            _, name, form, bits = ln.split("|")
            rows.append((name, form, tuple(ps.KEYS[int(b)] for b in bits.split(",") if b)))
    assert rows == [(name, form, tuple(k for k in ps.KEYS if k in refused)) for _, name, form, refused in ps.ROWS]


def _sources():
    return {f: open(os.path.join(CSRC, f)).read() for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh", ".h"))}


def test_no_refusal_macro_or_message_outside_the_table():
    """Refusals of the ten settings are written in plan_settings.h and formatted by refuse_settings only; the checks of other kinds
    (SKI, kernel sums, row sharding) keep their own words."""
    src = _sources()
    assert not [f for f, s in src.items() if "GP_REFUSE_" in s]
    check = re.search(r"int refuse_settings\(const gp_plan\* p, CallId call\) \{.*?\n\}\n", src["api.cu"], re.S).group(0)
    assert "is not available on %s (%s)" in check and "as a %s is not available (%s)" in check
    for f, s in src.items():
        if f == "plan_settings.h":
            continue
        s = s.replace(check, "")
        assert "is not available on %s (%s)" not in s and "as a factor is not available" not in s and "as a term is not available" not in s, f
        for _, noun, _ in ps.SETTINGS:
            assert f"is not available on {noun}" not in s and f"{noun} as a" not in s, (f, noun)


def test_every_refusal_the_sources_used_to_name_is_a_row():
    """The (call, setting) pairs the per-feature tests once found in the sources, as rows of the oracle."""
    pairs = {
        "additive": ["set_backend", "set_tasks", "set_kron", "set_sum", "set_product", "set_ski", "kmv_input_grad",
                     "kdense_input_grad", "set_deriv", "set_deriv_kind", "set_comm", "sum_term", "product_factor"],
        "periodic": ["set_tasks", "set_kron", "set_product", "set_ski", "set_sum", "set_additive", "set_spectral", "kmv_input_grad",
                     "kdense_input_grad", "set_deriv", "set_deriv_kind", "deriv_data", "kron_data", "product_factor", "set_comm"],
        "poly": ["set_additive", "set_periodic", "set_ski", "set_spectral", "set_tasks", "product_factor", "set_product", "set_kron",
                 "kron_data", "set_deriv", "deriv_data"],
        "spectral": ["set_backend", "set_tasks", "set_kron", "set_sum", "set_product", "set_ski", "set_additive", "kmv_input_grad",
                     "kdense_input_grad", "set_deriv", "set_deriv_kind", "set_comm", "sum_term", "product_factor", "kron_data",
                     "deriv_data"],
        "rq": ["set_tasks", "set_kron", "set_deriv", "set_deriv_kind", "set_product", "set_ski", "set_additive", "set_spectral",
               "set_periodic", "set_comm", "product_factor", "kron_data", "deriv_data", "kron_data_refresh"],
    }
    for setting, rows in pairs.items():
        for row in rows:
            assert ps.refused(row, (setting,)) == setting, (row, setting)
