"""The ctypes binding of the CPU oracle against oracle/oracle.h (no GPU): one checked declaration per exported function and
struct mirrors with a C compiler's layout.  ctypes passes a wrongly declared argument or a misplaced field as garbage without any
error, and every parity test trusts what the oracle computes."""
import os
import re
import subprocess

from oracle import oracle as O
from test_capi_symbols import ROOT, _header, check_prototypes, check_struct_layouts

HEADER = os.path.join(ROOT, "oracle", "oracle.h")
MIRRORS = {"oracle_view": O.OView, "oracle_params": O.OParams, "oracle_sgm_pixel": O.SGM_PIXEL, "oracle_dmap": O.ODMap}


def test_binding_prototypes_match_the_header():
	check_prototypes(HEADER, "oracle_", O.PROTOTYPES, MIRRORS)


def test_library_exports_exactly_the_declared_functions():
	"""An extern "C" function that oracle.h does not declare has no table entry and no compiler check of its definition."""
	declared = set(re.findall(r"\b(oracle_\w+)\s*\(", _header(HEADER)))
	out = subprocess.check_output(["nm", "-D", "--defined-only", O.build()], text=True)
	exported = {l.split()[-1] for l in out.splitlines() if l.split()[-1].startswith("oracle_")}
	assert exported == declared


def test_struct_layouts_match_a_c_compiler(tmp_path):
	got = check_struct_layouts(tmp_path, HEADER, MIRRORS)
	assert got["oracle_sgm_pixel"] == 16  # the records oracle_sgm_match shares with the engine's b200mvs_sgm_pixel
