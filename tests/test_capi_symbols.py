"""The C-ABI library builds, loads and exports every symbol include/b200mvs.h declares
(no compute calls: there is no GPU here)."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "b200mvs.h")


def _header(path=HEADER):
	"""a C header without comments"""
	return re.sub(r"/\*.*?\*/", "", open(path).read(), flags=re.S)


def _declared():
	return sorted(set(re.findall(r"\b(b200mvs_[a-z_0-9]+)\s*\(", _header())))


def _layout(mirror):
	"""(size, [(field, offset), ...]) of a ctypes Structure or of a numpy structured dtype"""
	if isinstance(mirror, type):
		return C.sizeof(mirror), [(f[0], getattr(mirror, f[0]).offset) for f in mirror._fields_]
	return mirror.itemsize, [(f, mirror.fields[f][1]) for f in mirror.names]


def check_struct_layouts(tmp_path, header, mirrors):
	"""sizeof / offsetof of every struct of `header` as gcc sees them == its mirror (struct name -> ctypes Structure or numpy
	structured dtype).  -> gcc's numbers, {"struct": size, "struct.field": offset}"""
	import subprocess
	lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "%s"' % os.path.basename(header), 'int main(void) {']
	for cname, m in mirrors.items():
		lines.append('printf("%s %%zu\\n", sizeof(%s));' % (cname, cname))
		for fname, _ in _layout(m)[1]:
			lines.append('printf("%s.%s %%zu\\n", offsetof(%s, %s));' % (cname, fname, cname, fname))
	lines.append('return 0; }')
	src = tmp_path/"layout.c"
	src.write_text("\n".join(lines))
	exe = str(tmp_path/"layout")
	subprocess.check_call(["gcc", "-std=c99", "-I", os.path.dirname(header), "-o", exe, str(src)])
	got = dict(l.split() for l in subprocess.check_output([exe], text=True).splitlines())
	for cname, m in mirrors.items():
		size, fields = _layout(m)
		assert int(got[cname]) == size, cname
		for fname, offset in fields:
			assert int(got["%s.%s" % (cname, fname)]) == offset, (cname, fname)
	return {k: int(v) for k, v in got.items()}


def check_prototypes(header, prefix, prototypes, mirrors):
	"""Every entry of `prototypes` (name -> (restype, argtypes), a ctypes binding's table) has the arity, argument types and return
	type of its prototype in `header`, one entry per function named `prefix`..., in header order.  mirrors: every struct the header
	defines -> its ctypes Structure (or the numpy dtype of records passed as arrays).  ctypes passes a wrongly declared argument as
	garbage without any error."""
	src = re.sub(r"^\s*#.*$", "", _header(header), flags=re.M)
	protos = re.findall(r"([\w\s*]+?)\b(%s\w+)\s*\(([^()]*)\)\s*;" % prefix, src)
	assert [name for _, name, _ in protos] == list(prototypes)  # one entry per prototype, in header order
	assert set(re.findall(r"}\s*(%s\w+)\s*;" % prefix, src)) == set(mirrors)
	scalars = {"int": C.c_int, "unsigned": C.c_uint, "float": C.c_float, "double": C.c_double, "long long": C.c_longlong,
		"uint64_t": C.c_uint64, "size_t": C.c_size_t, "uint8_t": C.c_uint8, "int16_t": C.c_int16, "uint16_t": C.c_uint16,
		"uint32_t": C.c_uint32}

	def allowed(words):
		"""ctypes types that pass the C type `words` (tokens without const and the parameter name) correctly"""
		stars = words.count("*")
		base = " ".join(w for w in words if w != "*")
		if stars == 0:
			return [None] if base == "void" else [scalars[base]]
		if stars > 1:
			return [C.POINTER(C.c_void_p)]
		if base == "char":
			return [C.c_char_p]
		if base in mirrors:
			return ([C.POINTER(mirrors[base])] if isinstance(mirrors[base], type) else []) + [C.c_void_p]
		return [C.c_void_p] + ([C.POINTER(scalars[base])] if base in scalars else [])

	tokens = lambda decl: [w for w in decl.replace("*", " * ").split() if w != "const"]
	# a parameter without its name; an array parameter (`float n[3]`) is the pointer it decays to
	param = lambda decl: tokens(decl)[:-1] + (["*"] if "[" in tokens(decl)[-1] else [])
	for ret, name, params in protos:
		restype, argtypes = prototypes[name]
		assert restype in allowed(tokens(ret)), (name, ret.strip())
		params = [] if params.strip() == "void" else [param(p) for p in params.split(",")]
		assert len(argtypes) == len(params), name
		for k, (words, t) in enumerate(zip(params, argtypes)):
			assert t in allowed(words), (name, k, " ".join(words))


def _mirrors():
	"""every struct of include/b200mvs.h -> its ctypes mirror in openmvs_b200/lib.py"""
	from openmvs_b200 import lib
	return {"b200mvs_view": lib.View, "b200mvs_params": lib.Params, "b200mvs_stats": lib.Stats, "b200mvs_job": lib.Job,
		"b200mvs_sgm_params": lib.SgmParams, "b200mvs_dmap": lib.DMap, "b200mvs_filter_params": lib.FilterParams,
		"b200mvs_debug": lib.Debug, "b200mvs_sgm_pixel": lib.SgmPixel, "b200mvs_fuse_view": lib.FuseView, "b200mvs_fuse_params": lib.FuseParams}


def test_library_builds_and_exports_every_declared_symbol():
	from openmvs_b200 import build, lib
	path = build.build_extension()
	assert os.path.exists(path)
	dll = C.CDLL(path)
	names = _declared()
	assert len(names) >= 21
	for n in names:
		assert hasattr(dll, n), "missing export %s" % n
	# the python binding lists exactly the declared symbols
	assert sorted(lib.SYMBOLS) == names


def test_struct_layouts_match_header_sizes():
	from openmvs_b200 import lib
	# b200mvs_view: pointer, 3 ints (+pad), 21 doubles, pointer, 3 ints (+pad), 21 doubles
	assert C.sizeof(lib.View) == 8+16+21*8+8+16+21*8-8+8 or C.sizeof(lib.View) % 8 == 0
	assert C.sizeof(lib.Params) == 19*4
	assert C.sizeof(lib.Stats) == 8+8+8+8+4+4+8+4+4


def test_struct_layouts_match_a_c_compiler(tmp_path):
	"""sizeof / offsetof of every struct of include/b200mvs.h as gcc sees them == the ctypes mirrors in openmvs_b200/lib.py"""
	got = check_struct_layouts(tmp_path, HEADER, _mirrors())
	assert got["b200mvs_sgm_pixel"] == 16  # SemiGlobalMatcher::PixelData


def test_binding_prototypes_match_the_header():
	"""Every entry of lib.PROTOTYPES has the arity, argument types and return type of its prototype in include/b200mvs.h"""
	from openmvs_b200 import lib
	assert lib.SYMBOLS == list(lib.PROTOTYPES)
	check_prototypes(HEADER, "b200mvs_", lib.PROTOTYPES, _mirrors())


def test_binding_constants_match_the_header():
	from openmvs_b200 import lib
	defines = dict(re.findall(r"^#define B200MVS_(\w+)\s+(\d+)", _header(), flags=re.M))
	kept = [n for n in defines if hasattr(lib, n)]
	assert {"ABI_VERSION", "SGM_MAX_LEVELS"} <= set(kept)
	for n in kept:
		assert getattr(lib, n) == int(defines[n]), n


def test_create_without_gpu_fails_loudly():
	import torch
	if torch.cuda.is_available():
		pytest.skip("GPU present")
	from openmvs_b200 import lib
	from openmvs_b200.depth_estimator import PatchMatchB200
	with pytest.raises(lib.B200MVSError):
		PatchMatchB200(0)
	dll = lib.load()
	assert dll.b200mvs_device_count() == 0
	ctx = C.c_void_p()
	assert dll.b200mvs_create(0, C.byref(ctx)) == 3  # B200MVS_ERR_NOGPU: never a CPU fallback
	assert not ctx


def test_sources_do_not_reference_the_oracle():
	"""The product package must not import, link or execute anything under oracle/."""
	pkg = os.path.join(ROOT, "openmvs_b200")
	for dp, _, files in os.walk(pkg):
		for f in files:
			if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
				txt = open(os.path.join(dp, f)).read()
				assert "liboracle" not in txt and "from oracle" not in txt and "import oracle" not in txt, f


def test_null_context_and_bad_arguments_return_status_codes():
	"""Error behaviour at the boundary: status codes, never a crash or exit()."""
	from openmvs_b200 import lib
	dll = lib.load()
	assert dll.b200mvs_set_params(None, None) == 1
	assert dll.b200mvs_set_debug(None, None) == 1 and dll.b200mvs_set_ignore_mask(None, None, 0, 0, 0, 0) == 1
	assert dll.b200mvs_get_schedule(None, 0, None, None) == 1
	assert dll.b200mvs_abi_version() == lib.ABI_VERSION
	# the library reports the struct sizes it was compiled with (checked against the bindings by lib.load())
	assert dll.b200mvs_sizeof(1) == C.sizeof(lib.Params) and dll.b200mvs_sizeof(99) == 0
	assert dll.b200mvs_destroy(None) == 1
	assert dll.b200mvs_estimate(None, None, 0, C.c_float(1), C.c_float(2), -1, None, None, None, None, None) == 1
	assert dll.b200mvs_sync(None, None) == 1
	assert dll.b200mvs_estimate_batch(None, 0, None, 0) == 1
	assert dll.b200mvs_sgm_match(None, None, None, None, 0, 0, None, C.c_uint64(0), None, None, None, None) == 1
	assert dll.b200mvs_last_error(None) == b"null context"
	assert dll.b200mvs_filter_depth_map(None, None, None, 0, None, C.c_float(0), C.c_float(1), None, None, None, None) == 1
	assert dll.b200mvs_filter_depth_map_device(None, None, None, 0, None, C.c_float(0), C.c_float(1), None, None, None, None, None, None) == 1
	assert dll.b200mvs_remove_small_segments(None, None, None, None, 0, 0, C.c_float(0.01), 100, None) == 1
	assert dll.b200mvs_gap_interpolation_device(None, None, None, None, 0, 0, C.c_float(0.01), 7, None) == 1


def test_set_debug_refuses_reserved_and_unknown_fields():
	"""The retired PatchMatch switches and wave-front tuning switches are reserved fields of b200mvs_debug: naming one (or an old
	name) is an error, not a silent no-op.  The check runs before any call into the library."""
	from openmvs_b200 import lib
	from openmvs_b200.depth_estimator import PatchMatchB200
	names = [f for f, _ in lib.Debug._fields_]
	assert names[:2] == ["reserved0", "reserved1"] and names[4] == "reserved2"
	assert names[5:12] == ["reserved%d" % i for i in range(3, 10)]
	retired = ("noTMA", "scalarTaps", "sweepFourCtas",
		"frontLayout", "frontSerial", "frontBlock", "frontLag", "frontCtas", "frontDepth", "frontSubCell")
	pm = PatchMatchB200.__new__(PatchMatchB200)   # no context: SetDebug must refuse the name before using one
	for k in ("reserved",) + tuple(names[:2]) + tuple(names[4:12]) + retired:
		with pytest.raises(AttributeError):
			pm.SetDebug(**{k: 1})
