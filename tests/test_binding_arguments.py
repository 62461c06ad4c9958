"""The buffer checks of the Python binding (depth_estimator._arg): every map, image and volume argument is checked for residency,
dtype, shape, layout and size before its address reaches the C-ABI, which can not check a raw pointer.

No case here lets a refused argument reach the library: the engine objects are built without a context (__new__), their device is
set by hand, and _call is a stub that records its arguments and stops the method there.  A refusal the binding misses therefore
fails an assertion; it never runs a kernel.  The CPU part runs without a GPU; the GPU part (-m gpu) only allocates tensors."""
import ctypes as C
import inspect
import re
from types import SimpleNamespace

import numpy as np
import pytest

from openmvs_b200 import depth_estimator as DE, lib
from openmvs_b200.depth_estimator import Camera, DepthData, DepthMapsData, PatchMatchB200, SemiGlobalMatcher, ViewData

torch = pytest.importorskip("torch")

H, W = 20, 30
NV = (H-6)*(W-6)     # pixel-map records of a W x H pair
N = 500              # numCosts
CAM = Camera(np.array([[30.0, 0, 15], [0, 30.0, 10], [0, 0, 1]]), np.eye(3), np.zeros(3))


class Reached(Exception):
	"""raised by the stub: the method got as far as a library call"""


class Stub:
	"""_Context._call: records (name, args) and stops the method, except for calls that pass no buffer"""
	PASS = ("set_params",)

	def __init__(self):
		self.calls = []

	def __call__(self, name, *args):
		self.calls.append((name, args))
		if name not in self.PASS:
			raise Reached("b200mvs_" + name)


def engines(device, monkeypatch=None):
	"""a PatchMatchB200, a SemiGlobalMatcher and a DepthMapsData without a context, on `device`, sharing one stub; with monkeypatch
	also the per-device contexts of the module-level calls"""
	stub = Stub()
	pm, sgm, ctx = PatchMatchB200.__new__(PatchMatchB200), SemiGlobalMatcher.__new__(SemiGlobalMatcher), DE._Context.__new__(DE._Context)
	for o in (pm, sgm, ctx):
		o.device, o._ctx, o._lib, o.stats, o._call = device, C.c_void_p(), lib.load(), lib.Stats(), stub
	pm.bGeomConsistency = False
	sgm.prm = lib.SgmParams(3, 4, 14.0, 38.0)
	dm = DepthMapsData.__new__(DepthMapsData)
	dm.pmCUDA, dm.nCalibratedImages, dm.stats, dm.arrDepthData = pm, 12, lib.Stats(), []
	if monkeypatch is not None:
		for index in range(max(torch.cuda.device_count(), 1)):
			monkeypatch.setitem(DE._DEVICE_CTX, index, ctx)
	return SimpleNamespace(pm=pm, sgm=sgm, dm=dm, stub=stub)


# ---- the table: every public call that passes a buffer address to the library --------------------------------------------
# argument kinds: FREE sets a size the call takes as given, TIED must match the size of another argument (COPY too, but a strided
# tensor is copied, not refused), VOL is a volume of at least N elements, REC a pixel map of 16-byte records, ANY a volume without a
# size the binding can know
FREE, TIED, COPY, VOL, REC, ANY = "free", "tied", "copied", "volume", "records", "any"
F32, I16, U8 = "float32", "int16", "uint8"


def Arg(dtype, shape, kind=FREE):
	return (dtype, shape, kind)


def _dd(a, depth="depthMap", conf="confMap"):
	return DepthData([ViewData(None, CAM)], 1.0, 2.0, depthMap=a[depth], confMap=a.get(conf))


def _views(a):
	return [ViewData(a["image"], CAM), ViewData(a["image"], CAM, depthMap=a.get("neighbourDepth"))]


_STATE = dict(image=Arg(F32, (H, W)), plane4=Arg(F32, (H, W, 4), TIED), cost=Arg(F32, (H, W), TIED), lowres=Arg(F32, (H, W), TIED))
_PAIR = dict(leftGray=Arg(F32, (H, W)), leftColor=Arg(U8, (H, W, 3), TIED), rightGray=Arg(F32, (H, W), TIED),
	rightColor=Arg(U8, (H, W, 3), TIED))
_INIT = SemiGlobalMatcher.HierarchyLevels(W, H, 0)[1]

# name -> (arguments, call(engines, arguments), whether the call has a host form that numpy maps take)
DEVICE = {
	"PatchMatchB200.ToGray": (dict(image=Arg(U8, (H, W, 3))), lambda e, a: e.pm.ToGray(a["image"]), False),
	"PatchMatchB200.ScaleImage": (dict(image=Arg(F32, (H, W))), lambda e, a: e.pm.ScaleImage(a["image"], 0.5), False),
	"PatchMatchB200.SetIgnoreMask": (dict(mask=Arg(U8, (H, W))), lambda e, a: e.pm.SetIgnoreMask(a["mask"]), True),
	"PatchMatchB200.EstimateDepthMap": (dict(image=Arg(F32, (H, W)), neighbourDepth=Arg(F32, (H, W)), depthMap=Arg(F32, (H, W), TIED),
		normalMap=Arg(F32, (H, W, 3), TIED), confMap=Arg(F32, (H, W), TIED), viewsMap=Arg(U8, (H, W, 4), TIED)),
		lambda e, a: e.pm.EstimateDepthMap(DepthData(_views(a), 1.0, 2.0, a["depthMap"], a["normalMap"], a["confMap"], a["viewsMap"])), True),
	"PatchMatchB200.ScoreDepthMap": (_STATE, lambda e, a: e.pm.ScoreDepthMap(_views(a), 1.0, 2.0, a["plane4"], a["cost"], a["lowres"]), False),
	"PatchMatchB200.SweepDepthMap": (_STATE, lambda e, a: e.pm.SweepDepthMap(_views(a), 1.0, 2.0, a["plane4"], a["cost"], 0, nRandomIters=3,
		lowres=a["lowres"]), False),
	"DepthMapsData.FilterDepthMap": (dict(depthMap=Arg(F32, (H, W)), confMap=Arg(F32, (H, W), TIED), nbDepth=Arg(F32, (H-2, W+4)),
		nbConf=Arg(F32, (H-2, W+4), TIED)), lambda e, a: e.dm.FilterDepthMap(_dd(a), [_dd(a, "nbDepth", "nbConf")], True), True),
	"DepthMapsData.RemoveSmallSegments": (dict(depthMap=Arg(F32, (H, W)), normalMap=Arg(F32, (H, W, 3), TIED), confMap=Arg(F32, (H, W), TIED)),
		lambda e, a: e.dm.RemoveSmallSegments(DepthData([], 0, 0, a["depthMap"], a["normalMap"], a["confMap"])), True),
	"DepthMapsData.GapInterpolation": (dict(depthMap=Arg(F32, (H, W)), normalMap=Arg(F32, (H, W, 3), TIED), confMap=Arg(F32, (H, W), TIED)),
		lambda e, a: e.dm.GapInterpolation(DepthData([], 0, 0, a["depthMap"], a["normalMap"], a["confMap"])), True),
	"SemiGlobalMatcher.MatchDevice": (dict(leftGray=Arg(F32, (H, W)), leftColor=Arg(U8, (H, W, 3), TIED), rightGray=Arg(F32, (H, W), TIED),
		imagePixels=Arg(U8, (NV, 16), REC), costs=Arg(U8, (N,), VOL), accums=Arg(I16, (N,), VOL)),
		lambda e, a: e.sgm.MatchDevice(a["leftGray"], a["leftColor"], a["rightGray"], a["imagePixels"], N, costs=a["costs"], accums=a["accums"]), False),
	"SemiGlobalMatcher.ConsistencyCrossCheck": (dict(l2r=Arg(I16, (H, W)), r2l=Arg(I16, (H, W), TIED)),
		lambda e, a: e.sgm.ConsistencyCrossCheck(a["l2r"], a["r2l"]), False),
	"SemiGlobalMatcher.RefineDisparityMap": (dict(disparityMap=Arg(I16, (H, W)), imagePixels=Arg(U8, (H*W, 16), REC), accums=Arg(I16, (N,), ANY)),
		lambda e, a: e.sgm.RefineDisparityMap(a["disparityMap"], a["imagePixels"], a["accums"]), False),
	"SemiGlobalMatcher.MatchPairDevice": (_PAIR, lambda e, a: e.sgm.MatchPairDevice(a["leftGray"], a["leftColor"], a["rightGray"],
		a["rightColor"], -16, 0, overlap=False), False),
	"SemiGlobalMatcher.MatchPairHierarchicalDevice": (dict(_PAIR, leftMask=Arg(U8, (H, W), TIED), rightMask=Arg(U8, (H, W), TIED),
		initDisparity=Arg(I16, (_INIT[1], _INIT[0]), TIED)), lambda e, a: e.sgm.MatchPairHierarchicalDevice(a["leftGray"], a["leftColor"],
		a["rightGray"], a["rightColor"], a["initDisparity"], a["leftMask"], a["rightMask"], minResolution=0), False),
	"SemiGlobalMatcher.Disparity2RangeMap": (dict(disparityMap=Arg(I16, (H, W)), maskMap=Arg(U8, (2*H+8, 2*W+8))),
		lambda e, a: e.sgm.Disparity2RangeMap(a["disparityMap"], a["maskMap"]), False),
	"SemiGlobalMatcher.FlipDirection": (dict(l2r=Arg(I16, (H, W))), lambda e, a: e.sgm.FlipDirection(a["l2r"]), False),
	"SemiGlobalMatcher.UpscaleMask": (dict(maskMap=Arg(U8, (H, W))), lambda e, a: e.sgm.UpscaleMask(a["maskMap"], (2*W+6, 2*H+6)), False),
	"SemiGlobalMatcher.ExtractMask": (dict(disparityMap=Arg(I16, (H, W)), maskMap=Arg(U8, (H, W), TIED)),
		lambda e, a: e.sgm.ExtractMask(a["disparityMap"], a["maskMap"]), False),
	"SemiGlobalMatcher.FilterSpeckles": (dict(disparityMap=Arg(I16, (H, W))), lambda e, a: e.sgm.FilterSpeckles(a["disparityMap"]), False),
	"SemiGlobalMatcher.ResizeAreaU8": (dict(image=Arg(U8, (H, W, 3))), lambda e, a: e.sgm.ResizeAreaU8(a["image"], 2), False),
	"SemiGlobalMatcher.LevelMask": (dict(mask=Arg(U8, (H, W))), lambda e, a: e.sgm.LevelMask(a["mask"], (W//2, H//2)), False),
	"SemiGlobalMatcher.ProjectDisparity2DepthMap": (dict(disparityMap=Arg(I16, (H, W)), costMap=Arg(I16, (H, W), TIED)),
		lambda e, a: e.sgm.ProjectDisparity2DepthMap(a["disparityMap"], a["costMap"], np.eye(4), 4, (W, H)), False),
	"SemiGlobalMatcher.Fuse": (dict(disparity=Arg(I16, (H, W)), cost=Arg(I16, (H, W), TIED)),
		lambda e, a: e.sgm.Fuse([(a["disparity"], a["cost"], np.eye(4), 4)], (W, H)), True),
	"EstimateNormalMap": (dict(depthMap=Arg(F32, (H, W))), lambda e, a: DE.EstimateNormalMap(np.eye(3), a["depthMap"]), False),
	"FuseDepthMaps": (dict(depth=Arg(F32, (H, W)), normal=Arg(F32, (H, W, 3), COPY), conf=Arg(F32, (H, W), COPY), color=Arg(U8, (H, W, 3), COPY)),
		lambda e, a: DE.FuseDepthMaps([dict(a, K=CAM.K, R=CAM.R, C=CAM.C)]), True),
}
MODULE_LEVEL = {"EstimateNormalMap", "FuseDepthMaps"}   # run on a context of the tensors' own device


def _maps(*shapes, dtype=np.float32):
	return [None if s is None else np.zeros(s, dtype) for s in shapes]


def _read_only(shape):
	a = np.zeros(shape, np.float32)
	a.flags.writeable = False
	return a


HOST = {
	# name -> [(refused call(engines), what is wrong), ...]
	"DepthMapsData.RemoveSmallSegments": [
		(lambda e: e.dm.RemoveSmallSegments(DepthData([], 0, 0, *_maps((H, W), (H, W), None))), "normal map without its 3 channels"),
		(lambda e: e.dm.RemoveSmallSegments(DepthData([], 0, 0, *_maps((H, W), None, (H, W+1)))), "confidence map of another size"),
		(lambda e: e.dm.RemoveSmallSegments(DepthData([], 0, 0, np.zeros((H, W)))), "float64 depth map")],
	"DepthMapsData.GapInterpolation": [
		(lambda e: e.dm.GapInterpolation(DepthData([], 0, 0, *_maps((H, W), (H, W), None))), "normal map without its 3 channels"),
		(lambda e: e.dm.GapInterpolation(DepthData([], 0, 0, *_maps((H, W), None, (H-1, W)))), "confidence map of another size"),
		(lambda e: e.dm.GapInterpolation(DepthData([], 0, 0, np.zeros((H, W))[:, ::2])), "strided float64 depth map")],
	"DepthMapsData.FilterDepthMap": [
		(lambda e: e.dm.FilterDepthMap(_dd(dict(zip(("depthMap", "confMap"), _maps((H, W), (H, W-1))))), []), "reference confidence map of another size"),
		(lambda e: e.dm.FilterDepthMap(_dd(dict(zip(("depthMap", "confMap"), _maps((H, W), (H, W))))),
			[_dd(dict(zip(("depthMap", "confMap"), _maps((H, W), (W, H)))))], True), "neighbour confidence map of another size")],
	"PatchMatchB200.EstimateDepthMap": [
		(lambda e: e.pm.EstimateDepthMap(DepthData(_views(dict(image=np.zeros((H, W), np.float32))), 1.0, 2.0, normalMap=np.zeros((H, W)))),
			"normal map without its 3 channels"),
		(lambda e: e.pm.EstimateDepthMap(DepthData(_views(dict(image=np.zeros((H, W)))), 1.0, 2.0)), "float64 image")],
	"EstimateDepthMapsBatch": [
		(lambda e: DE.EstimateDepthMapsBatch([DepthData(_views(dict(image=torch.zeros(H, W))), 1.0, 2.0)], [e.pm]), "tensor images"),
		(lambda e: DE.EstimateDepthMapsBatch([DepthData(_views(dict(image=np.zeros((H, W), np.float32))), 1.0, 2.0,
			viewsMap=np.zeros((H, W, 3), np.uint8))], [e.pm]), "views map with 3 entries per pixel")],
	"PatchMatchB200.SetIgnoreMask": [(lambda e: e.pm.SetIgnoreMask(np.zeros((H, W, 1))), "3-D mask")],
	"SemiGlobalMatcher.Match": [
		(lambda e: e.sgm.Match(*_maps((H, W)), np.zeros((H, W), np.uint8), *_maps((H, W)), np.zeros((NV, 16), np.uint8), N), "gray colour image"),
		(lambda e: e.sgm.Match(*_maps((H, W)), np.zeros((H, W, 3), np.uint8), *_maps((H, W)), np.zeros((NV-1, 16), np.uint8), N),
			"pixel map one record short"),
		(lambda e: e.sgm.Match(*_maps((H, W)), np.zeros((H, W, 3), np.uint8), *_maps((H, W+2)), np.zeros((NV, 16), np.uint8), N),
			"right image of another size")],
	"SemiGlobalMatcher.Fuse": [
		(lambda e: e.sgm.Fuse([(np.zeros((H, W), np.int16), np.zeros((H, W-1), np.uint16), np.eye(4), 4)], (W, H)), "cost map of another size"),
		(lambda e: e.sgm.Fuse([(np.zeros(H*W, np.int16), None, np.eye(4), 4)], (W, H)), "1-D disparity map")],
	"SemiGlobalMatcher.PairQ": [(lambda e: SemiGlobalMatcher.PairQ(np.eye(3), *([np.eye(3), np.eye(3), np.zeros(3)]*2)), "3 x 3 Q")],
	"FuseDepthMaps": [
		(lambda e: DE.FuseDepthMaps([dict(depth=np.zeros((H, W)), K=CAM.K, R=CAM.R, C=CAM.C)]), "float64 depth map"),
		(lambda e: DE.FuseDepthMaps([dict(depth=np.zeros((H, W), np.float32), normal=np.zeros((H, W)), K=CAM.K, R=CAM.R, C=CAM.C)]),
			"normal map without its 3 channels"),
		(lambda e: DE.FuseDepthMaps([dict(depth=_read_only((H, W)), K=CAM.K, R=CAM.R, C=CAM.C)]), "read-only depth map")],
}
# public calls that pass only arrays they allocate themselves
OWN_BUFFERS = {"FuseRoundStats"}


# ---- coverage guard ----------------------------------------------------------------------------------------------------------
_ADDRESS = re.compile(r"data_ptr\(\)|\.ctypes\.data\b|\b_arg\(")


def _passing_buffers():
	"""qualified names of the public methods (PatchMatchB200, SemiGlobalMatcher, DepthMapsData) and module-level functions whose
	source, or the source of a private helper they call, passes a buffer address to the library"""
	src = {}
	for scope in (DE, DE._Context, PatchMatchB200, DepthMapsData, SemiGlobalMatcher):
		for f in vars(scope).values():
			f = getattr(f, "__func__", f)
			if inspect.isfunction(f) and f.__module__ == DE.__name__:
				src[f.__qualname__] = inspect.getsource(f)
	bare = lambda q: q.rsplit(".", 1)[-1]
	passing = {q for q, s in src.items() if _ADDRESS.search(s)}
	while True:
		helpers = {bare(q) for q in passing if bare(q).startswith("_")}
		more = {q for q, s in src.items() if q not in passing and helpers & set(re.findall(r"\b(_\w+)\(", s))}
		if not more:
			return {q for q in passing if not bare(q).startswith("_")}
		passing |= more


def test_every_call_that_passes_a_buffer_has_a_case():
	passing = _passing_buffers()
	assert {"SemiGlobalMatcher.MatchDevice", "DepthMapsData.RemoveSmallSegments", "PatchMatchB200.EstimateDepthMap", "FuseDepthMaps",
		"EstimateDepthMapsBatch"} <= passing, sorted(passing)
	missing = passing - set(DEVICE) - set(HOST) - OWN_BUFFERS
	assert not missing, "calls that pass buffers to the library without a case here: %s" % sorted(missing)


# ---- CPU part ------------------------------------------------------------------------------------------------------------------
def _make(args, where, dtype=None):
	"""valid arguments as zeroed CUDA tensors (where = "cuda:i"), CPU tensors ("cpu") or numpy arrays ("numpy")"""
	out = {}
	for name, (dt, shape, _) in args.items():
		t = torch.zeros(shape, dtype=getattr(torch, dt))
		out[name] = t.numpy() if where == "numpy" else t.to(where)
	return out


@pytest.mark.parametrize("name", sorted(DEVICE))
def test_device_calls_refuse_host_memory(name, monkeypatch):
	args, call, host_form = DEVICE[name]
	forms = ["cpu"] + ([] if host_form else ["numpy"])
	for where in forms:
		e = engines(0, monkeypatch)
		with pytest.raises(ValueError):
			call(e, _make(args, where))
		assert not e.stub.calls, (where, e.stub.calls)


@pytest.mark.parametrize("name", sorted(HOST))
def test_host_calls_refuse_malformed_maps(name, monkeypatch):
	for call, what in HOST[name]:
		e = engines(0, monkeypatch)
		with pytest.raises(ValueError):
			call(e)
		assert not e.stub.calls, (what, e.stub.calls)


def _addresses(args):
	"""every address among the arguments of a call: integers and the pointer fields of the structs it passes"""
	out = set()
	for a in args:
		a = a.contents if isinstance(a, C._Pointer) else getattr(a, "_obj", a)
		for s in (a if isinstance(a, C.Array) else [a]):
			if isinstance(s, C.Structure):
				out |= {getattr(s, f) for f, t in s._fields_ if t is C.c_void_p}
			elif isinstance(s, int):
				out.add(s)
	return out


@pytest.mark.parametrize("name", sorted(n for n, (_, _, host_form) in DEVICE.items() if host_form and n not in MODULE_LEVEL))
def test_valid_host_calls_pass_the_arrays_in_place(name, monkeypatch):
	"""the host form of a call takes numpy maps of the right dtype as they are: their own addresses reach the library"""
	args, call, _ = DEVICE[name]
	a = _make(args, "numpy")
	if name == "SemiGlobalMatcher.Fuse":
		a["cost"] = a["cost"].view(np.uint16)
	e = engines(0, monkeypatch)
	with pytest.raises(Reached):
		call(e, a)
	fn, passed = e.stub.calls[-1]
	assert not [k for k, v in a.items() if v.ctypes.data not in _addresses(passed)], fn


def test_valid_sgm_host_match_passes_the_arrays_in_place(monkeypatch):
	e = engines(0, monkeypatch)
	a = [np.zeros((H, W), np.float32), np.zeros((H, W, 3), np.uint8), np.zeros((H, W), np.float32), np.zeros((NV, 16), np.uint8)]
	with pytest.raises(Reached):
		e.sgm.Match(*a, N)
	fn, passed = e.stub.calls[-1]
	assert fn == "sgm_match" and [passed[0], passed[1], passed[2], passed[5]] == [x.ctypes.data for x in a]


def test_refusals_name_the_method_the_argument_and_both_shapes(monkeypatch):
	e = engines(0, monkeypatch)
	with pytest.raises(ValueError) as err:
		e.dm.RemoveSmallSegments(DepthData([], 0, 0, *_maps((H, W), (H, W), None)))
	msg = str(err.value)
	assert msg.startswith("RemoveSmallSegments: normalMap must be") and "(%d, %d, 3)" % (H, W) in msg and "(%d, %d)" % (H, W) in msg


# ---- GPU part ------------------------------------------------------------------------------------------------------------------
WRONG = {F32: ("float16", "float64"), I16: ("int32", "float16"), U8: ("int32",)}


def _mutations(dtype, shape, kind, dev):
	"""(what, a refused form of one argument) on device dev"""
	z = lambda s, dt=dtype: torch.zeros(s, dtype=getattr(torch, dt), device=dev)
	yield "numpy", z(shape).cpu().numpy()
	yield "cpu tensor", z(shape).cpu()
	if torch.cuda.device_count() > 1:
		yield "other device", z(shape).to("cuda:%d" % (1-torch.device(dev).index))
	for dt in WRONG[dtype]:
		yield dt, z(shape, dt)
	if kind != COPY:
		yield "column stride 2", z(shape[:-1]+(2*shape[-1],))[..., ::2]
	if kind in (FREE, TIED, COPY):
		yield "extra dimension", z(shape+(1,))
	if kind in (TIED, COPY):
		yield "one row short", z((shape[0]-1,)+shape[1:])
	if kind in (VOL, REC):
		yield "one %s short" % ("record" if kind == REC else "element"), z((shape[0]-1,)+shape[1:])


def _cuda():
	if not torch.cuda.is_available():
		pytest.skip("no CUDA device")


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(DEVICE))
def test_device_calls_accept_valid_tensors_and_refuse_each_malformed_argument(name, monkeypatch):
	_cuda()
	args, call, host_form = DEVICE[name]
	e = engines(0, monkeypatch)
	with pytest.raises(Reached):
		call(e, _make(args, "cuda:0"))
	for arg, spec in args.items():
		for what, bad in _mutations(*spec, "cuda:0"):
			if what == "numpy" and host_form and len(args) == 1:
				continue    # the host form of the call
			if what == "other device" and name in MODULE_LEVEL and len(args) == 1:
				continue    # runs on the context of the tensor's device
			a = _make(args, "cuda:0")
			a[arg] = bad
			e = engines(0, monkeypatch)
			with pytest.raises(ValueError):
				call(e, a)
			assert not e.stub.calls, (arg, what, e.stub.calls)


@pytest.mark.gpu
@pytest.mark.parametrize("tensors", [0, 1])
@pytest.mark.parametrize("name", sorted(set(DEVICE) - MODULE_LEVEL))
def test_device_calls_refuse_tensors_of_another_device_than_the_context(name, tensors, monkeypatch):
	"""tensors on cuda:0 for a context recorded on device 1 (the index is set by hand, so this runs on one GPU: the call is refused
	before anything touches device 1), and with two GPUs tensors on cuda:1 for a context on device 0"""
	_cuda()
	if tensors >= torch.cuda.device_count():
		pytest.skip("needs two GPUs")
	args, call, _ = DEVICE[name]
	e = engines(1-tensors, monkeypatch)
	with pytest.raises(ValueError):
		call(e, _make(args, "cuda:%d" % tensors))
	assert not e.stub.calls
