"""Host-side mirror of the reference interface of the hot path.

Names, argument meaning and error behaviour follow the reference so that the parity tests
read like tests of the reference:

  OPTDENSE            option namespace              libs/MVS/DepthMap.cpp:69-114
  Camera              K, R, C                       libs/MVS/Camera.h
  ViewData, DepthData in/out container              libs/MVS/DepthMap.h:157-271
  PatchMatchB200      the PatchMatchCUDA seam       libs/MVS/PatchMatchCUDA.inl:78-131
                      (ctor(device), Init(bGeomConsistency), Release(), EstimateDepthMap(DepthData&))
  DepthMapsData       EstimateDepthMap(idxImage, nGeometricIter)   libs/MVS/SceneDensify.cpp:616-805
                      FilterDepthMap / RemoveSmallSegments / GapInterpolation   libs/MVS/SceneDensify.cpp:810-1299

Everything here is plumbing above the C-ABI (include/b200mvs.h); the arithmetic runs in the
CUDA kernels of openmvs_b200/csrc.  numpy arrays take the host path (H2D/D2H inside the
call, like the reference seam); torch CUDA tensors take the device-resident path.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import math
from typing import List, Optional

import numpy as np

from . import lib as _lib


class OPTDENSE:
	"""The OPTDENSE knobs the estimator consumes, with the reference defaults
	(libs/MVS/DepthMap.cpp:69-114).  Class attributes, like the reference's globals."""
	nSubResolutionLevels = 2
	nNumViews = 0
	nEstimationIters = 3
	nEstimationGeometricIters = 2
	fEstimationGeometricWeight = 0.1
	nRandomIters = 6
	fNCCThresholdKeep = 0.9
	fDescriptorMinMagnitudeThreshold = 0.02
	fRandomDepthRatio = 0.003
	fRandomAngle1Range = 16.0
	fRandomAngle2Range = 10.0
	fRandomSmoothDepth = 0.02
	fRandomSmoothNormal = 13.0
	fRandomSmoothBonus = 0.93
	# depth-map post-processing (FilterDepthMap / RemoveSmallSegments / GapInterpolation)
	nMinViewsFilter = 2
	nMinViewsFilterAdjust = 1
	bFilterAdjust = True
	fDepthDiffThreshold = 0.01
	nSpeckleSize = 100
	nIpolGapSize = 7
	# engine schedule (not in the reference; include/b200mvs.h b200mvs_params): 0 = automatic number of red-black sweeps
	nSweepsPerIter = 0
	nPropagation = 4
	nPropagationFar = 2
	bSkipUnchanged = 1
	nEvalCap = 0
	nSeed = 1234

	@classmethod
	def schedule(cls, geometric: bool = False):
		"""(red-black sweeps, refinement tries per sweep) the engine runs for the current options (b200mvs_get_schedule)."""
		n, r = C.c_int(), C.c_int()
		p = cls.snapshot()
		_lib.load().b200mvs_get_schedule(C.byref(p), int(bool(geometric)), C.byref(n), C.byref(r))
		return n.value, r.value

	@classmethod
	def snapshot(cls) -> _lib.Params:
		p = _lib.Params()
		for name, _ in _lib.Params._fields_:
			if name == "seed":
				p.seed = cls.nSeed
			else:
				setattr(p, name, getattr(cls, name))
		return p


@dataclasses.dataclass
class Camera:
	K: np.ndarray
	R: np.ndarray
	C: np.ndarray


@dataclasses.dataclass
class ViewData:
	"""DepthData::ViewData: gray float image in [0,1] + camera (+ known depth-map and its camera)."""
	image: object            # (H, W) float32 gray image, or the (H, W, 3|4) uint8 colour image (converted on the device); numpy or torch CUDA
	camera: Camera
	depthMap: object = None  # optional (H, W) float32
	cameraDepthMap: Optional[Camera] = None
	bgr: bool = True         # channel order of a uint8 colour image: B,G,R as cv::imread delivers (False: R,G,B)


@dataclasses.dataclass
class DepthData:
	images: List[ViewData]   # reference view first
	dMin: float
	dMax: float
	depthMap: object = None
	normalMap: object = None
	confMap: object = None
	viewsMap: object = None

	def IsValid(self) -> bool:
		return len(self.images) > 0

	def IsEmpty(self) -> bool:
		return self.depthMap is None

	def Save(self, fileName: str, IDs=None, imageFileName: str = "image.jpg") -> bool:
		"""DepthData::Save (libs/MVS/DepthMap.cpp:237-251): write depth/normal/conf/views as a .dmap file."""
		from . import dmap_io
		tonp = lambda a: None if a is None else (a.detach().cpu().numpy() if _is_torch(a) else np.asarray(a))
		ref = self.images[0]
		h, w = tonp(self.depthMap).shape
		ids = list(IDs) if IDs is not None else list(range(len(self.images)))
		return dmap_io.ExportDepthDataRaw(fileName, imageFileName, ids, (w, h), ref.camera.K, ref.camera.R, ref.camera.C,
			self.dMin, self.dMax, tonp(self.depthMap), tonp(self.normalMap), tonp(self.confMap), tonp(self.viewsMap))

	def Load(self, fileName: str, flags: int = 15) -> bool:
		"""DepthData::Load: read the maps and the depth range back from a .dmap file."""
		from . import dmap_io
		d = dmap_io.ImportDepthDataRaw(fileName, flags)
		self.depthMap, self.normalMap, self.confMap, self.viewsMap = d["depthMap"], d["normalMap"], d["confMap"], d["viewsMap"]
		self.dMin, self.dMax = d["dMin"], d["dMax"]
		return True


def _stream_handle(device) -> int:
	"""cudaStream_t of torch's current stream.  The C-ABI treats NULL as "use the context's own
	stream", so torch's legacy default stream (handle 0) is passed as cudaStreamLegacy (0x1)."""
	import torch
	h = torch.cuda.current_stream(device).cuda_stream
	return h if h else 1


def _is_torch(a) -> bool:
	return type(a).__module__.startswith("torch")


def _cuda_index(a) -> int:
	"""the CUDA device of a tensor, which the module-level device calls run on (0 for anything else: the checks then refuse it)"""
	return a.device.index if _is_torch(a) and a.is_cuda else 0


def _pitch(a) -> int:
	"""row pitch in bytes of a numpy array or a torch tensor"""
	return a.stride(0)*a.element_size() if _is_torch(a) else a.strides[0]


def _host(a, dtype, device=None):
	"""a map in the form the host calls take it: a C-contiguous numpy array of dtype, copied only if it has to be.  A map for a
	device call (device given), a CUDA tensor and None are returned as they are, for _arg to judge."""
	return a if device is not None or a is None or (_is_torch(a) and a.is_cuda) else np.ascontiguousarray(a, dtype)


# a 16-bit volume or cost map: the library reads uint16, which torch callers often hold as int16
_U16 = ("int16", "uint16")


def _arg(where: str, name: str, a, dtype, shape=None, device=None, rows: bool = False, min_size: int = 0):
	"""Check one buffer argument of a library call -> its address (None for None, the C-ABI's "not given").  A raw pointer carries
	no size, type or device, so this is the only place that can refuse a buffer the call would overrun, misread or fault on.
	dtype: a dtype name or a tuple of names; an int: the byte size of the records of a pixel map, whose `shape` then counts records.
	shape: the exact shape with None for any size and a tuple for a choice of sizes; None: any shape.
	device: None for a numpy array (host call), else the index of the CUDA device the tensor must be on.
	rows: every row contiguous, rows may be strided; else C-contiguous.  min_size: the least number of elements (volumes).
	Raises ValueError naming the method, the argument, what was expected and what was given.  Reads attributes only: no
	synchronisation, no copy."""
	if a is None:
		return None
	tensor = _is_torch(a)
	if tensor:
		kind, item, resident = str(a.dtype)[len("torch."):], a.element_size(), a.is_cuda and a.device.index == device
		steps = [s*item for s in a.stride()]
	elif isinstance(a, np.ndarray):
		kind, item, steps, resident = a.dtype.name, a.itemsize, a.strides, device is None
	else:
		kind, item, steps, resident = type(a).__name__, 0, (), False
	dims = tuple(getattr(a, "shape", ()))
	size = math.prod(dims)
	if isinstance(dtype, int):
		typed, counted = size*item % dtype == 0, (size*item//dtype,)
	else:
		typed, counted = kind in ((dtype,) if isinstance(dtype, str) else dtype), dims
	packed = all(n == 1 or s == item*math.prod(dims[k+1:]) for k, (n, s) in enumerate(zip(dims, steps)) if k or not rows)
	fits = shape is None or (len(counted) == len(shape) and all(
		s is None or (n in s if isinstance(s, tuple) else n == s) for n, s in zip(counted, shape)))
	if resident and typed and packed and fits and size >= min_size:
		return a.data_ptr() if tensor else a.ctypes.data
	layout = "row-contiguous" if rows else "contiguous"
	sizes = lambda s: "(%s)" % ", ".join("*" if n is None else "|".join(map(str, n)) if isinstance(n, tuple) else str(n) for n in s)
	want = "a %s %s" % (layout, "numpy array" if device is None else "CUDA tensor on cuda:%d" % device)
	if isinstance(dtype, int):
		want += " of %s records of %d bytes" % (shape[0], dtype)
	else:
		want += " of %s" % "|".join((dtype,) if isinstance(dtype, str) else dtype)
		want += "" if shape is None else " of shape %s" % sizes(shape)
	want += " of at least %d elements" % min_size if min_size else ""
	home = "tensor on %s" % a.device if tensor else "numpy array" if isinstance(a, np.ndarray) else "object"
	raise ValueError("%s: %s must be %s; got a %s %s of shape %s%s" % (where, name, want, kind, home, sizes(dims),
		"" if packed else ", not " + layout))


def _put_camera(o, cam: Camera, suffix: str = ""):
	for name in ("K", "R", "C"):
		getattr(o, name+suffix)[:] = np.asarray(getattr(cam, name), np.float64).ravel()


def _make_views(images: List[ViewData], device: Optional[int] = None, where: str = "EstimateDepthMap"):
	"""-> (ctypes View array, keepalive list, on_device flag).  Tensor views must be CUDA tensors on `device` (None: numpy views only)."""
	arr = (_lib.View*len(images))()
	keep = []
	dev = _is_torch(images[0].image)
	home = device if dev else None
	for i, v in enumerate(images):
		o = arr[i]
		img = v.image if _is_torch(v.image) else np.asarray(v.image)
		keep.append(img)
		if str(img.dtype).endswith("uint8"):
			# 8-bit colour image with packed pixels (Image8U3): toGray runs on the device inside the call
			o.image8 = _arg(where, "images[%d].image" % i, img, "uint8", (None, None, (3, 4)), home, rows=True)
			o.height, o.width, o.channels8 = img.shape; o.stride8_bytes = _pitch(img); o.bgr8 = int(bool(v.bgr))
		else:
			o.image = _arg(where, "images[%d].image" % i, img, "float32", (None, None), home, rows=True)
			o.height, o.width = img.shape; o.stride_bytes = _pitch(img)
		_put_camera(o, v.camera)
		if v.depthMap is not None and i > 0:
			dm = _host(v.depthMap, np.float32, home)
			o.depth = _arg(where, "images[%d].depthMap" % i, dm, "float32", (None, None), home, rows=True)
			keep.append(dm)
			o.dheight, o.dwidth = dm.shape; o.dstride_bytes = _pitch(dm)
			_put_camera(o, v.cameraDepthMap or v.camera, "d")
	return arr, keep, dev


# the output maps of a DepthData: (name, channels, dtype)
_MAPS = (("depthMap", (), "float32"), ("normalMap", (3,), "float32"), ("confMap", (), "float32"), ("viewsMap", (4,), "uint8"))


def _out_maps(dd: DepthData, device: Optional[int] = None, where: str = "EstimateDepthMap"):
	"""Check the given output maps of dd (converted numpy arrays for a host call, CUDA tensors on `device` for a device call), then
	allocate the missing ones zeroed -> the four addresses."""
	h, w = dd.images[0].image.shape[:2]
	maps = [(name, (h, w)+ch, dt, _host(getattr(dd, name), dt, device)) for name, ch, dt in _MAPS]
	for name, shape, dt, a in maps:
		_arg(where, name, a, dt, shape, device)
	ptrs = []
	for name, shape, dt, a in maps:
		if a is None and device is None:
			a = np.zeros(shape, dt)
		elif a is None:
			import torch
			a = torch.zeros(shape, dtype=getattr(torch, dt), device=device)
		setattr(dd, name, a)
		ptrs.append(_arg(where, name, a, dt, shape, device))
	return ptrs


def _host_maps(dd: DepthData, where: str = "EstimateDepthMap"):
	"""_out_maps of a host call: numpy output maps -> their addresses"""
	return _out_maps(dd, None, where)


class _Context:
	"""One engine context (b200mvs_create ... b200mvs_destroy) on CUDA device `device`, and the calls made on it."""

	def __init__(self, device: int):
		self.device = int(device)
		self._lib = _lib.load()
		self._ctx = C.c_void_p()
		rc = self._lib.b200mvs_create(int(device), C.byref(self._ctx))
		if rc != 0:
			raise _lib.B200MVSError("b200mvs_create(device=%d) failed with status %d (no GPU => no fallback)" % (device, rc))
		self.stats = _lib.Stats()

	def _call(self, name: str, *args):
		"""b200mvs_<name>(ctx, *args); a non-zero status raises B200MVSError with the context's last error."""
		fn = "b200mvs_" + name
		_lib.check(self._lib, self._ctx, getattr(self._lib, fn)(self._ctx, *args), fn)

	def Release(self):
		if self._ctx:
			self._lib.b200mvs_destroy(self._ctx)
			self._ctx = C.c_void_p()

	def __del__(self):
		try:
			self.Release()
		except Exception:
			pass

	def SetDebug(self, **kw):
		"""b200mvs_set_debug: diagnostic kernel switches, the fields of b200mvs_debug; no arguments = defaults.
		SGM: sgmAggregation (0 auto, 1 general, 2 register-pipelined uniform, 3 bulk-copy ring, 4 wave fronts) and sgmCost
		(0 auto, 1 SIMT, 2 tensor cores).  PatchMatch has no switches.
		An unknown or reserved field name raises AttributeError."""
		d = _lib.Debug()
		for k, v in kw.items():
			if k.startswith("reserved") or not hasattr(d, k):
				raise AttributeError(k)
			setattr(d, k, int(v))
		self._call("set_debug", C.byref(d))


class PatchMatchB200(_Context):
	"""Drop-in for the reference's `PatchMatchCUDA` (libs/MVS/PatchMatchCUDA.inl:78-131)."""

	def __init__(self, device: int = 0):
		super().__init__(device)
		self.bGeomConsistency = False

	def Init(self, bGeomConsistency: bool = False):
		"""PatchMatchCUDA::Init: select photometric (false) or geometric-consistency (true) passes."""
		self.bGeomConsistency = bool(bGeomConsistency)

	def ToGray(self, image, bgr: bool = True):
		"""TImage::toGray(out, COLOR_BGR2GRAY, bNormalize=true) (libs/Common/Types.inl:2377-2431) on the device: uint8 CUDA tensor
		(H, W, 3|4), channel order B,G,R(,A) as cv::imread delivers (bgr=False: R,G,B) -> float32 gray (H, W) in [0, 1]."""
		import torch
		ptr = _arg("ToGray", "image", image, "uint8", (None, None, (3, 4)), self.device)
		h, w, ch = (int(v) for v in image.shape)
		out = torch.empty((h, w), dtype=torch.float32, device=image.device)
		self._call("to_gray_device", ptr, w, h, w*ch, ch, int(bool(bgr)), out.data_ptr(), w*4, _stream_handle(self.device))
		return out

	def ScaleImage(self, image, scale: float):
		"""DepthData::ViewData::ScaleImage (libs/MVS/DepthMap.h:193-203) on the device: float32 CUDA tensor (H, W) ->
		cv::resize(image, Size(), scale, scale, scale > 1 ? INTER_CUBIC : INTER_AREA), or None when |scale - 1| < 0.15
		(the reference keeps the image then)."""
		import torch
		ptr = _arg("ScaleImage", "image", image, "float32", (None, None), self.device, rows=True)
		h, w = (int(v) for v in image.shape)
		dw, dh, ok = C.c_int(), C.c_int(), C.c_int()
		self._lib.b200mvs_scaled_size(w, h, scale, C.byref(dw), C.byref(dh))
		out = torch.empty((max(dh.value, 1), max(dw.value, 1)), dtype=torch.float32, device=image.device)
		self._call("scale_image_device", ptr, w, h, _pitch(image), scale, out.data_ptr(), C.byref(ok), _stream_handle(self.device))
		return out if ok.value else None

	def _set_params(self):
		self._call("set_params", C.byref(OPTDENSE.snapshot()))

	def SetIgnoreMask(self, mask=None):
		"""Ignore-mask of the reference view for the following EstimateDepthMap calls (OPTDENSE::nIgnoreMaskLabel >= 0,
		libs/MVS/DepthMap.cpp:215-230,300-323): (H, W) uint8, 0 = ignored; numpy array (copied) or torch CUDA tensor
		(kept by reference until cleared); None clears it."""
		self._mask_keep = None
		if mask is None:
			self._call("set_ignore_mask", None, 0, 0, 0, 0)
			return
		home = self.device if _is_torch(mask) else None
		m = _host(mask, np.uint8, home)
		ptr = _arg("SetIgnoreMask", "mask", m, "uint8", (None, None), home, rows=True)
		if home is not None:
			self._mask_keep = m
		self._call("set_ignore_mask", ptr, int(m.shape[1]), int(m.shape[0]), _pitch(m), int(home is not None))

	def EstimateDepthMap(self, depthData: DepthData, nGeometricIter: Optional[int] = None, stream=None, sync: bool = True):
		"""PatchMatchCUDA::EstimateDepthMap(DepthData&): estimate depthMap/normalMap/confMap/viewsMap
		of depthData in place.  nGeometricIter defaults to -1 (photometric) or 0 (after Init(true))."""
		if not depthData.IsValid() or len(depthData.images) < 2:
			raise ValueError("DepthData needs the reference view and at least one neighbour")
		if nGeometricIter is None:
			nGeometricIter = 0 if self.bGeomConsistency else -1
		arr, keep, dev = _make_views(depthData.images, self.device)
		maps = _out_maps(depthData, self.device if dev else None)
		self._set_params()
		job = (arr, len(arr), depthData.dMin, depthData.dMax, int(nGeometricIter))
		if dev:
			if stream is None:
				stream = _stream_handle(self.device)
			self._call("estimate_device", *job, *maps, stream, C.byref(self.stats) if sync else None)
		elif sync:
			self._call("estimate", *job, *maps, C.byref(self.stats))
		else:
			# asynchronous host path: the caller keeps depthData alive and calls Wait() before reading the maps
			self._call("estimate_async", *job, *maps)
			self._inflight = (depthData, keep)
		return depthData

	def Wait(self):
		"""b200mvs_sync: wait for an EstimateDepthMap(..., sync=False) on host buffers and fetch its stats."""
		self._call("sync", C.byref(self.stats))
		self._inflight = None

	# ---- building blocks on device tensors (used by the parity tests) -----------------------
	def _state(self, where, images, plane4, cost, lowres):
		"""the device views and the float32 state of their reference image (H, W) -> (views, keepalive, [lowres, plane4, cost addresses])"""
		arr, keep, dev = _make_views(images, self.device, where)
		if not dev:
			raise ValueError("%s: building blocks need device-resident views" % where)
		h, w = images[0].image.shape[:2]
		return arr, keep, [_arg(where, name, a, "float32", shape, self.device)
			for name, a, shape in (("lowres", lowres, (h, w)), ("plane4", plane4, (h, w, 4)), ("cost", cost, (h, w)))]

	def ScoreDepthMap(self, images, dMin, dMax, plane4, cost, lowres=None):
		"""pass A (ScoreDepthMapTmp) on a packed plane field (H, W, 4) = {nx,ny,nz,depth}."""
		arr, keep, (lr, p4, c) = self._state("ScoreDepthMap", images, plane4, cost, lowres)
		self._set_params()
		self._call("pm_score", arr, len(arr), dMin, dMax, lr, p4, c, _stream_handle(self.device))

	def SweepDepthMap(self, images, dMin, dMax, plane4, cost, sweep, half=-1, nRandomIters=None, lowres=None):
		"""pass B: one red-black sweep (both colours, or one if half in {0,1})."""
		arr, keep, (lr, p4, c) = self._state("SweepDepthMap", images, plane4, cost, lowres)
		self._set_params()
		if nRandomIters is None:
			nRandomIters = OPTDENSE.schedule()[1]
		self._call("pm_sweep", arr, len(arr), dMin, dMax, lr, int(sweep), int(half), int(nRandomIters), p4, c, _stream_handle(self.device))


def EstimateDepthMapsBatch(arrDepthData: List[DepthData], engines: List["PatchMatchB200"], nGeometricIter: int = -1):
	"""b200mvs_estimate_batch: estimate every DepthData (host buffers) with the given engines — one per GPU of
	the box, or two on one GPU — dealt round-robin inside this process."""
	lib = engines[0]._lib
	jobs = (_lib.Job*len(arrDepthData))()
	keep = []
	for j, dd in enumerate(arrDepthData):
		arr, k, _ = _make_views(dd.images, None, "EstimateDepthMapsBatch")   # host buffers only
		keep.append((arr, k))
		J = jobs[j]
		J.views = arr; J.nViews = len(arr); J.dMin = dd.dMin; J.dMax = dd.dMax; J.nGeometricIter = int(nGeometricIter)
		J.depth, J.normal, J.conf, J.viewsMap = _host_maps(dd, "EstimateDepthMapsBatch")
	for e in engines:
		e._set_params()
	ctxs = (C.c_void_p*len(engines))(*[e._ctx for e in engines])
	rc = lib.b200mvs_estimate_batch(ctxs, len(engines), jobs, len(arrDepthData))
	if rc != 0:
		bad = [j for j in range(len(arrDepthData)) if jobs[j].status]
		raise _lib.B200MVSError("b200mvs_estimate_batch: jobs %s failed with status %d" % (bad, rc))
	return arrDepthData


class DepthMapsData:
	"""The slice of the reference's DepthMapsData around the hot path (libs/MVS/SceneDensify.h:52-93):
	arrDepthData + EstimateDepthMap(idxImage, nGeometricIter), and the per-view post-processing that
	follows it: RemoveSmallSegments, GapInterpolation, FilterDepthMap (SceneDensify.cpp:810-1299)."""

	def __init__(self, arrDepthData: List[DepthData], device: int = 0, nCalibratedImages: Optional[int] = None):
		self.arrDepthData = arrDepthData
		self.pmCUDA = PatchMatchB200(device)
		self.nCalibratedImages = len(arrDepthData) if nCalibratedImages is None else int(nCalibratedImages)
		self.stats = _lib.Stats()

	def EstimateDepthMap(self, idxImage: int, nGeometricIter: int = -1) -> bool:
		self.pmCUDA.Init(nGeometricIter >= 0)
		self.pmCUDA.EstimateDepthMap(self.arrDepthData[idxImage], nGeometricIter)
		return True

	@staticmethod
	def _dmap(o: "_lib.DMap", depthData: DepthData, need_conf: bool, keep: list, device: Optional[int], label: str):
		"""fill o with the depth and confidence maps of depthData: host maps (device None) are converted to float32, device maps
		must be CUDA tensors on `device` -> the depth map"""
		d, c = _host(depthData.depthMap, np.float32, device), _host(depthData.confMap, np.float32, device)
		if need_conf and c is None:
			raise ValueError("FilterDepthMap needs the confidence map of every view")
		o.depth = _arg("FilterDepthMap", label+".depthMap", d, "float32", (None, None), device)
		o.conf = _arg("FilterDepthMap", label+".confMap", c, "float32", tuple(d.shape), device)
		keep += [d, c]
		o.height, o.width = int(d.shape[0]), int(d.shape[1])
		_put_camera(o, depthData.images[0].camera)
		return d

	def FilterDepthMap(self, depthDataRef: DepthData, neighbors: List[DepthData], bAdjust: Optional[bool] = None, projected: bool = False):
		"""DepthMapsData::FilterDepthMap(depthDataRef, idxNeighbors, bAdjust) (SceneDensify.cpp:1050-1299).
		`neighbors` are the DepthData of the (at most 8, SceneDensify.cpp:2152) neighbour views whose depth-maps are valid.
		Returns (newDepthMap, newConfMap) — what the reference saves as filtered.dmap / filtered.cmap — or None when the map
		can not be filtered; with projected=True also the N projected neighbour depth and confidence maps (device path)."""
		bAdjust = OPTDENSE.bFilterAdjust if bAdjust is None else bool(bAdjust)
		prm = _lib.FilterParams(min(OPTDENSE.nMinViewsFilter, self.nCalibratedImages-1),
			min(OPTDENSE.nMinViewsFilterAdjust, self.nCalibratedImages-1), OPTDENSE.fDepthDiffThreshold, int(bAdjust))
		arr = (_lib.DMap*(len(neighbors)+1))()
		keep: list = []
		device = self.pmCUDA.device if _is_torch(depthDataRef.depthMap) else None
		dref = self._dmap(arr[0], depthDataRef, True, keep, device, "depthDataRef")
		for i, nb in enumerate(neighbors):
			self._dmap(arr[i+1], nb, bAdjust, keep, device, "neighbors[%d]" % i)
		nbrs = C.cast(C.byref(arr, C.sizeof(_lib.DMap)), C.POINTER(_lib.DMap))
		ok = C.c_int(0)
		if device is not None:
			import torch
			od = torch.empty_like(dref); oc = torch.empty_like(dref)
			pd = pc = None
			if projected:
				pd = torch.empty((max(len(neighbors), 1),)+tuple(dref.shape), dtype=torch.float32, device=dref.device)
				pc = torch.zeros_like(pd)
			self.pmCUDA._call("filter_depth_map_device", C.byref(arr[0]), nbrs, len(neighbors), C.byref(prm), depthDataRef.dMin,
				depthDataRef.dMax, od.data_ptr(), oc.data_ptr(), pd.data_ptr() if projected else None,
				pc.data_ptr() if projected and bAdjust else None, C.byref(ok), _stream_handle(device))
			if not ok.value:
				return None
			return (od, oc, pd, pc) if projected else (od, oc)
		od = np.empty_like(dref); oc = np.empty_like(dref)
		self.pmCUDA._call("filter_depth_map", C.byref(arr[0]), nbrs, len(neighbors), C.byref(prm), depthDataRef.dMin, depthDataRef.dMax,
			od.ctypes.data, oc.ctypes.data, C.byref(ok), C.byref(self.stats))
		return (od, oc) if ok.value else None

	def _post(self, where: str, name: str, depthData: DepthData, arg: int) -> bool:
		"""one in-place pass over the float32 maps of depthData: numpy arrays (host form) or CUDA tensors on pmCUDA's device"""
		d = depthData.depthMap
		device = self.pmCUDA.device if _is_torch(d) else None
		pd = _arg(where, "depthMap", d, "float32", (None, None), device)
		h, w = int(d.shape[0]), int(d.shape[1])
		pn = _arg(where, "normalMap", depthData.normalMap, "float32", (h, w, 3), device)
		pc = _arg(where, "confMap", depthData.confMap, "float32", (h, w), device)
		if device is not None:
			self.pmCUDA._call(name+"_device", pd, pn, pc, w, h, OPTDENSE.fDepthDiffThreshold, int(arg), _stream_handle(device))
		else:
			self.pmCUDA._call(name, pd, pn, pc, w, h, OPTDENSE.fDepthDiffThreshold, int(arg), C.byref(self.stats))
		return True

	def RemoveSmallSegments(self, depthData: DepthData) -> bool:
		"""DepthMapsData::RemoveSmallSegments (SceneDensify.cpp:810-900), depthData's maps in place."""
		return self._post("RemoveSmallSegments", "remove_small_segments", depthData, OPTDENSE.nSpeckleSize)

	def GapInterpolation(self, depthData: DepthData) -> bool:
		"""DepthMapsData::GapInterpolation (SceneDensify.cpp:904-1045), depthData's maps in place."""
		return self._post("GapInterpolation", "gap_interpolation", depthData, OPTDENSE.nIpolGapSize)


class SemiGlobalMatcher(_Context):
	"""The pair matcher of the reference's STEREO::SemiGlobalMatcher
	(libs/MVS/SemiGlobalMatcher.h:61-203): Match(left, right) -> (disparityMap, costMap) over the
	valid region, with the ctor parameters P1, P2, P2alpha, P2beta (defaults 3, 4, 14, 38)."""
	NO_DISP = 32767
	NO_ACCUMCOST = 65535

	def __init__(self, P1: int = 3, P2: int = 4, P2alpha: float = 14.0, P2beta: float = 38.0, device: int = 0):
		super().__init__(device)
		self.prm = _lib.SgmParams(int(P1), int(P2), float(P2alpha), float(P2beta))

	def Release(self):
		if getattr(self, "_peer", None) is not None:
			self._peer.Release(); self._peer = None
		super().Release()

	def Match(self, leftGray, leftColor, rightGray, imagePixels, numCosts: int):
		"""Host path: numpy images (gray float32 HxW, colour uint8 HxWx3 BGR) and the PixelMap
		(structured array from synth.sgm_pixel_map or any {u8 idx, i2 dmin, i2 dmax, i4} records)."""
		lg, lc, rg, px = _host(leftGray, np.float32), _host(leftColor, np.uint8), _host(rightGray, np.float32), _host(imagePixels, None)
		(h, w), (plg, plc, prg, _) = self._images("Match", lg, lc, rg, None, None)
		ppx = _arg("Match", "imagePixels", px, 16, ((w-6)*(h-6),))
		disp = np.zeros((h-6, w-6), np.int16); cost = np.zeros((h-6, w-6), np.uint16)
		self._call("sgm_match", plg, plc, prg, w, h, ppx, numCosts, C.byref(self.prm), disp.ctypes.data, cost.ctypes.data, C.byref(self.stats))
		return disp, cost

	def _images(self, where, leftGray, leftColor, rightGray, rightColor, device):
		"""check the rectified images of a match: gray float32 (h, w), colour uint8 (h, w, 3) -> ((h, w), their addresses)"""
		plg = _arg(where, "leftGray", leftGray, "float32", (None, None), device)
		h, w = (int(n) for n in leftGray.shape)
		return (h, w), [plg] + [_arg(where, name, a, dt, shape, device) for name, a, dt, shape in (("leftColor", leftColor, "uint8", (h, w, 3)),
			("rightGray", rightGray, "float32", (h, w)), ("rightColor", rightColor, "uint8", (h, w, 3)))]

	def MatchDevice(self, leftGray, leftColor, rightGray, imagePixels, numCosts: int, stages: int = 7, costs=None, accums=None, sync: bool = True):
		"""Device-resident path on torch CUDA tensors; costs (uint8) / accums (uint16 viewed as int16)
		are optional in/out volumes of numCosts entries.  Returns (disparity, cost) int16 tensors
		(cost holds the uint16 bit pattern)."""
		import torch
		(h, w), (plg, plc, prg, _) = self._images("MatchDevice", leftGray, leftColor, rightGray, None, self.device)
		ppx = _arg("MatchDevice", "imagePixels", imagePixels, 16, ((w-6)*(h-6),), self.device)
		pcv = _arg("MatchDevice", "costs", costs, "uint8", None, self.device, min_size=numCosts)
		pac = _arg("MatchDevice", "accums", accums, _U16, None, self.device, min_size=numCosts)
		dev = leftGray.device
		disp = torch.zeros((h-6, w-6), dtype=torch.int16, device=dev)
		cost = torch.zeros((h-6, w-6), dtype=torch.int16, device=dev)
		self._call("sgm_match_device", plg, plc, prg, w, h, ppx, numCosts, C.byref(self.prm), int(stages), pcv, pac, disp.data_ptr(),
			cost.data_ptr(), _stream_handle(self.device), C.byref(self.stats) if sync else None)
		return disp, cost

	def ConsistencyCrossCheck(self, l2r, r2l, thCross: int = 1):
		"""SemiGlobalMatcher::ConsistencyCrossCheck on int16 CUDA tensors; l2r is modified in place."""
		pl = _arg("ConsistencyCrossCheck", "l2r", l2r, "int16", (None, None), self.device)
		h, w = l2r.shape
		pr = _arg("ConsistencyCrossCheck", "r2l", r2l, "int16", (h, w), self.device)
		self._call("sgm_cross_check_device", pl, pr, w, h, int(thCross), _stream_handle(self.device))
		return l2r

	def RefineDisparityMap(self, disparityMap, imagePixels, accums=None, subpixelSteps: int = 4):
		"""SemiGlobalMatcher::RefineDisparityMap (LC-blend) on CUDA tensors: the int16 disparityMap in place, the pixel map of its
		pixels and the 16-bit accumulated costs (None: those of the last match with this pixel map on the context)."""
		pd = _arg("RefineDisparityMap", "disparityMap", disparityMap, "int16", (None, None), self.device)
		ppx = _arg("RefineDisparityMap", "imagePixels", imagePixels, 16, (disparityMap.numel(),), self.device)
		pac = _arg("RefineDisparityMap", "accums", accums, _U16, None, self.device)
		self._call("sgm_refine_device", ppx, pac, pd, disparityMap.numel(), int(subpixelSteps), _stream_handle(self.device))
		return disparityMap

	def MatchPairDevice(self, leftGray, leftColor, rightGray, rightColor, minDisp: int, maxDisp: int, thCross: int = 1, subpixelSteps: int = 4,
			overlap: bool = True):
		"""The per-level body of SemiGlobalMatcher::Match(scene, ...) for one global range (non-tSGM branch,
		libs/MVS/SemiGlobalMatcher.cpp:643-725) on CUDA tensors: right->left match with the range [minDisp, maxDisp),
		left->right match with the mirrored range, cross-check of the left map, sub-pixel refinement.
		Returns (leftDisparity * subpixelSteps, rightDisparity) as int16 tensors (NO_DISP = 32767).
		overlap (default): the two matches run on two contexts / streams (they are independent until the cross-check), so the
		aggregation kernels of the two share the SMs."""
		import torch
		(h, w), _ = self._images("MatchPairDevice", leftGray, leftColor, rightGray, rightColor, self.device)
		nv = (w-6)*(h-6)
		num = int(maxDisp-minDisp)
		dev = leftGray.device
		def pixel_map(lo, hi):
			# PixelData{u64 idx; i16 dmin, dmax; i32 pad} of a dense volume with one range, built on the device and kept: 16 B per
			# pixel would otherwise be generated and uploaded for every pair (33 MB at 1080p)
			key = (nv, num, int(lo), int(hi), str(dev))
			cache = self.__dict__.setdefault("_pxmaps", {})
			if key not in cache:
				if len(cache) > 8:
					cache.clear()
				rec = torch.empty((nv, 2), dtype=torch.int64, device=dev)
				rec[:, 0] = torch.arange(nv, dtype=torch.int64, device=dev)*num
				rec[:, 1] = (int(lo) & 0xFFFF) | ((int(hi) & 0xFFFF) << 16)       # little endian: dmin, dmax, pad = 0
				cache[key] = rec.view(torch.uint8).reshape(nv, 16)
			return cache[key]
		# Match(rightDataLevel, leftDataLevel): the right image plays "left" with range [minDisp, maxDisp)
		pxr = pixel_map(minDisp, maxDisp)
		# ranges are mirrored for the left->right match (SemiGlobalMatcher.cpp:677-682)
		pxl = pixel_map(-maxDisp, -minDisp)
		if not overlap:
			rdisp, _ = self.MatchDevice(rightGray, rightColor, leftGray, pxr, nv*num)
			ldisp, _ = self.MatchDevice(leftGray, leftColor, rightGray, pxl, nv*num)
		else:
			if getattr(self, "_peer", None) is None:
				self._peer = SemiGlobalMatcher(device=self.device)
				self._peer.prm = self.prm
				self._side = torch.cuda.Stream(device=dev)
			main = torch.cuda.current_stream(dev)
			self._side.wait_stream(main)
			with torch.cuda.stream(self._side):
				rdisp, _ = self._peer.MatchDevice(rightGray, rightColor, leftGray, pxr, nv*num, sync=False)
				for t in (rightGray, rightColor, leftGray, pxr, rdisp):
					t.record_stream(self._side)
			ldisp, _ = self.MatchDevice(leftGray, leftColor, rightGray, pxl, nv*num, sync=False)
			main.wait_stream(self._side)
		self.ConsistencyCrossCheck(ldisp, rdisp, thCross)
		self.RefineDisparityMap(ldisp, pxl, None, subpixelSteps)  # accumulated costs of the last (left) match
		torch.cuda.current_stream(dev).synchronize()
		return ldisp, rdisp

	@staticmethod
	def HierarchyLevels(width: int, height: int, minResolution: int = 320):
		"""Level sizes of the hierarchical matcher, coarsest first, and the size of its initial disparity map (b200mvs_sgm_levels):
		([(w, h), ...], (initWidth, initHeight)).  Host arithmetic, no GPU needed."""
		lib = _lib.load()
		n, iw, ih = C.c_int(), C.c_int(), C.c_int()
		ws, hs = (C.c_int*_lib.SGM_MAX_LEVELS)(), (C.c_int*_lib.SGM_MAX_LEVELS)()
		rc = lib.b200mvs_sgm_levels(int(width), int(height), int(minResolution), C.byref(n), ws, hs, C.byref(iw), C.byref(ih))
		if rc != 0:
			raise _lib.B200MVSError("b200mvs_sgm_levels(%d, %d, %d) failed with status %d" % (width, height, minResolution, rc))
		return [(ws[k], hs[k]) for k in range(n.value)], (iw.value, ih.value)

	def MatchPairHierarchicalDevice(self, leftGray, leftColor, rightGray, rightColor, initDisparity=None, leftMask=None, rightMask=None,
			minResolution: int = 320, thCross: int = 1, subpixelSteps: int = 4, nSpeckleSize: Optional[int] = None):
		"""SemiGlobalMatcher::Match(scene, ...) for one rectified pair (libs/MVS/SemiGlobalMatcher.cpp:583-718) on CUDA tensors:
		the image pyramid, per level FlipDirection + Disparity2RangeMap + right->left and left->right matches, the first level's
		cross-checks, speckle filter and mask extraction, the later levels' cross-check, and the final sub-pixel refinement.
		initDisparity: int16 map of HierarchyLevels' init size in half-coarsest-level pixels (None: no estimate, NO_DISP);
		leftMask / rightMask: uint8 full-resolution masks (0 = invalid).  minResolution = 0: one level with the initial map's range.
		Returns (leftDisparity * subpixelSteps, cost, levels) with levels = [{"size": (w, h), "numCosts": (right, left)}, ...];
		cost holds the uint16 bit pattern in an int16 tensor."""
		import torch
		where = "MatchPairHierarchicalDevice"
		(h, w), images = self._images(where, leftGray, leftColor, rightGray, rightColor, self.device)
		masks = [_arg(where, name, m, "uint8", (h, w), self.device) for name, m in (("leftMask", leftMask), ("rightMask", rightMask))]
		sizes, (iw, ih) = self.HierarchyLevels(w, h, minResolution)
		pinit = _arg(where, "initDisparity", initDisparity, "int16", (ih, iw), self.device)
		dev = leftGray.device
		disp = torch.empty((h-6, w-6), dtype=torch.int16, device=dev)
		cost = torch.empty((h-6, w-6), dtype=torch.int16, device=dev)
		nums = (C.c_uint64*(2*len(sizes)))()
		speckle = OPTDENSE.nSpeckleSize if nSpeckleSize is None else nSpeckleSize
		self._call("sgm_match_hierarchical_device", *images, w, h, pinit, iw, ih, *masks, int(minResolution), int(speckle), int(thCross),
			int(subpixelSteps), C.byref(self.prm), disp.data_ptr(), cost.data_ptr(), nums, _stream_handle(self.device))
		levels = [{"size": sizes[k], "numCosts": (int(nums[2*k]), int(nums[2*k+1]))} for k in range(len(sizes))]
		return disp, cost, levels

	# building blocks of the level loop on CUDA tensors (names of the reference's members, SemiGlobalMatcher.h:171-179)
	def Disparity2RangeMap(self, disparityMap, maskMap, minNumDisp: int = 3, minNumDispInvalid: int = 16):
		"""-> (PixelMap as a (maskH*maskW, 16) uint8 tensor, numCosts) for the 2x grid of maskMap (int16 / uint8 tensors)"""
		import torch
		pd = _arg("Disparity2RangeMap", "disparityMap", disparityMap, "int16", (None, None), self.device)
		pm = _arg("Disparity2RangeMap", "maskMap", maskMap, "uint8", (None, None), self.device)
		h, w = disparityMap.shape
		mh, mw = maskMap.shape
		px = torch.empty((mh*mw, 16), dtype=torch.uint8, device=disparityMap.device)
		num = C.c_uint64()
		self._call("sgm_range_map_device", pd, w, h, pm, mw, mh, int(minNumDisp), int(minNumDispInvalid), px.data_ptr(), C.byref(num),
			_stream_handle(self.device))
		return px, int(num.value)

	def FlipDirection(self, l2r):
		"""-> the right->left int16 map of a left->right one"""
		import torch
		pl = _arg("FlipDirection", "l2r", l2r, "int16", (None, None), self.device)
		h, w = l2r.shape
		r2l = torch.empty_like(l2r)
		self._call("sgm_flip_direction_device", pl, r2l.data_ptr(), w, h, _stream_handle(self.device))
		return r2l

	def UpscaleMask(self, maskMap, size2x):
		"""-> the uint8 mask of size2x = (width, height)"""
		import torch
		pm = _arg("UpscaleMask", "maskMap", maskMap, "uint8", (None, None), self.device)
		h, w = maskMap.shape
		out = torch.empty((int(size2x[1]), int(size2x[0])), dtype=torch.uint8, device=maskMap.device)
		self._call("sgm_upscale_mask_device", pm, w, h, out.data_ptr(), int(size2x[0]), int(size2x[1]), _stream_handle(self.device))
		return out

	def ExtractMask(self, disparityMap, maskMap, thValid: int = 3):
		"""maskMap (uint8, same size) in place"""
		pd = _arg("ExtractMask", "disparityMap", disparityMap, "int16", (None, None), self.device)
		h, w = disparityMap.shape
		pm = _arg("ExtractMask", "maskMap", maskMap, "uint8", (h, w), self.device)
		self._call("sgm_extract_mask_device", pd, pm, w, h, int(thValid), _stream_handle(self.device))
		return maskMap

	def FilterSpeckles(self, disparityMap, newVal: int = NO_DISP, maxSpeckleSize: Optional[int] = None, maxDiff: int = 5):
		"""cv::filterSpeckles on an int16 tensor, in place; maxSpeckleSize defaults to OPTDENSE.nSpeckleSize"""
		pd = _arg("FilterSpeckles", "disparityMap", disparityMap, "int16", (None, None), self.device)
		h, w = disparityMap.shape
		size = OPTDENSE.nSpeckleSize if maxSpeckleSize is None else maxSpeckleSize
		self._call("sgm_filter_speckles_device", pd, w, h, int(newVal), int(size), int(maxDiff), _stream_handle(self.device))
		return disparityMap

	def ResizeAreaU8(self, image, factor: int):
		"""cv::resize(image, Size(), 1/factor, 1/factor, INTER_AREA) of a uint8 (H, W[, C]) tensor with 1, 3 or 4 channels"""
		import torch
		pi = _arg("ResizeAreaU8", "image", image, "uint8", (None, None) if len(image.shape) == 2 else (None, None, (1, 3, 4)), self.device)
		h, w = image.shape[:2]
		cn = 1 if image.dim() == 2 else image.shape[2]
		dh, dw = int(np.rint(h/float(factor))), int(np.rint(w/float(factor)))
		out = torch.empty((dh, dw) + tuple(image.shape[2:]), dtype=torch.uint8, device=image.device)
		self._call("resize_area_u8_device", pi, w, h, int(cn), int(factor), out.data_ptr(), _stream_handle(self.device))
		return out

	def LevelMask(self, mask, levelSize):
		"""first level's mask: NEAREST resize of the uint8 mask to levelSize = (w, h), cropped to the valid region"""
		import torch
		pm = _arg("LevelMask", "mask", mask, "uint8", (None, None), self.device)
		h, w = mask.shape
		lw, lh = int(levelSize[0]), int(levelSize[1])
		out = torch.empty((lh-6, lw-6), dtype=torch.uint8, device=mask.device)
		self._call("sgm_level_mask_device", pm, w, h, lw, lh, out.data_ptr(), _stream_handle(self.device))
		return out

	# fusion-mode -2: the disparity maps of the pairs that contain an image, projected into it and fused (SemiGlobalMatcher::Fuse,
	# libs/MVS/SemiGlobalMatcher.cpp:739-859)
	@staticmethod
	def PairQ(Q, Kleft, Rleft, Cleft, K, R, C):
		"""b200mvs_sgm_pair_q: the Q of a pair whose left image is the other view (camera Kleft, Rleft, Cleft), re-targeted to the image
		of camera (K, R, C), as Fuse does for the file <other>_<this>.dimap.  Host arithmetic, no GPU needed -> (4, 4) float64"""
		lib = _lib.load()
		arrs = [np.ascontiguousarray(a, np.float64).ravel() for a in (Q, Kleft, Rleft, Cleft, K, R, C)]
		if [a.size for a in arrs] != [16, 9, 9, 3, 9, 9, 3]:
			raise ValueError("Q must be 4x4, the K and R 3x3 and the C 3-vectors")
		out = np.zeros(16, np.float64)
		rc = lib.b200mvs_sgm_pair_q(*[a.ctypes.data for a in arrs], out.ctypes.data)
		if rc != 0:
			raise _lib.B200MVSError("b200mvs_sgm_pair_q failed with status %d (a zero focal length in Kleft)" % rc)
		return out.reshape(4, 4)

	def _pairs(self, pairs, device: bool, where: str = "Fuse"):
		"""[(disparity, cost or None, Q, subpixelSteps), ...] -> (ctypes b200mvs_sgm_pair array, keepalive list).  Host maps are
		converted to int16 / uint16; device maps must be CUDA tensors on the context's device."""
		if not 1 <= len(pairs) <= _lib.SGM_MAX_PAIRS:
			raise ValueError("%s: between 1 and %d pairs" % (where, _lib.SGM_MAX_PAIRS))
		home = self.device if device else None
		arr = (_lib.SgmPair*len(pairs))()
		keep = []
		for k, (o, (disp, cost, Q, steps)) in enumerate(zip(arr, pairs)):
			disp, cost = _host(disp, np.int16, home), _host(cost, np.uint16, home)
			o.disparity = _arg(where, "pairs[%d] disparity" % k, disp, "int16", (None, None), home)
			o.cost = _arg(where, "pairs[%d] cost" % k, cost, _U16, tuple(disp.shape), home)
			keep += [disp, cost]
			o.height, o.width = (int(x) for x in disp.shape)
			o.subpixelSteps = int(steps)
			o.Q[:] = list(np.asarray(Q, np.float64).reshape(16))
		return arr, keep

	def ProjectDisparity2DepthMap(self, disparityMap, costMap, Q, subpixelSteps: int, size):
		"""SemiGlobalMatcher::ProjectDisparity2DepthMap (SemiGlobalMatcher.cpp:1925-2039) of one pair on CUDA tensors (disparityMap
		int16, costMap 16-bit or None) into an image of size = (W, H) -> (depth (H, W), depthRange (H, W, 2), conf (H, W)) float32
		tensors; rejected pixels are 0 in all three, conf is 0 without a cost map."""
		import torch
		W, H = int(size[0]), int(size[1])
		arr, keep = self._pairs([(disparityMap, costMap, Q, subpixelSteps)], True, "ProjectDisparity2DepthMap")
		dev = disparityMap.device
		depth = torch.empty((H, W), dtype=torch.float32, device=dev)
		rng = torch.empty((H, W, 2), dtype=torch.float32, device=dev)
		conf = torch.empty((H, W), dtype=torch.float32, device=dev)
		self._call("sgm_project_disparity_device", arr, W, H, depth.data_ptr(), rng.data_ptr(), conf.data_ptr(), _stream_handle(self.device))
		return depth, rng, conf

	def Fuse(self, pairs, size, minViews: int = 2, K=None):
		"""SemiGlobalMatcher::Fuse (SemiGlobalMatcher.cpp:739-859) for one image of size = (W, H): pairs = [(disparity, cost or None,
		Q, subpixelSteps), ...] in the order the reference walks the image's neighbours, Q already re-targeted to this image (PairQ
		for pairs whose left image is the neighbour).  numpy maps take the host path, CUDA tensors the device path.
		K (3x3, optional): also EstimateNormalMap of the result (nEstimateNormals == 2).  -> (depth, conf, normal or None)"""
		W, H = int(size[0]), int(size[1])
		device = _is_torch(pairs[0][0]) if pairs else False
		arr, keep = self._pairs(pairs, device)
		k = None if K is None else np.ascontiguousarray(K, np.float64).reshape(9)
		kp = None if k is None else k.ctypes.data
		if device:
			import torch
			dev = pairs[0][0].device
			depth = torch.empty((H, W), dtype=torch.float32, device=dev)
			conf = torch.empty((H, W), dtype=torch.float32, device=dev)
			normal = torch.empty((H, W, 3), dtype=torch.float32, device=dev) if k is not None else None
			self._call("sgm_fuse_device", arr, len(pairs), W, H, int(minViews), kp, depth.data_ptr(), conf.data_ptr(),
				normal.data_ptr() if normal is not None else None, _stream_handle(self.device))
		else:
			depth = np.zeros((H, W), np.float32); conf = np.zeros((H, W), np.float32)
			normal = np.zeros((H, W, 3), np.float32) if k is not None else None
			self._call("sgm_fuse", arr, len(pairs), W, H, int(minViews), kp, depth.ctypes.data, conf.ctypes.data,
				normal.ctypes.data if normal is not None else None, C.byref(self.stats))
		return depth, conf, normal


_DEVICE_CTX = {}


def _device_context(dev) -> _Context:
	"""the context kept per device (a torch device or an index) for the module-level calls (EstimateNormalMap, FuseDepthMaps, the
	point-cloud calls; their host-buffer forms use device 0's)"""
	index = dev if isinstance(dev, int) else dev.index
	ctx = _DEVICE_CTX.get(index)
	if ctx is None:
		ctx = _DEVICE_CTX[index] = _Context(index)
	return ctx


def EstimateNormalMap(K, depthMap):
	"""MVS::EstimateNormalMap(K, depthMap, normalMap) (libs/MVS/DepthMap.cpp:1522-1613) on a float32 CUDA tensor -> (H, W, 3) unit
	camera-space normals (0 where undetermined).  K: 3x3, converted to float as the reference's Matrix3x3f argument.  Runs on a
	context kept per device."""
	import torch
	ptr = _arg("EstimateNormalMap", "depthMap", depthMap, "float32", (None, None), _cuda_index(depthMap))
	ctx = _device_context(depthMap.device)
	k = np.ascontiguousarray(K, np.float64).reshape(9)
	h, w = depthMap.shape
	normal = torch.empty((h, w, 3), dtype=torch.float32, device=depthMap.device)
	ctx._call("estimate_normal_map_device", ptr, w, h, k.ctypes.data, normal.data_ptr(), _stream_handle(ctx.device))
	return normal


@dataclasses.dataclass
class PointCloud:
	"""MVS::PointCloud as FuseDepthMaps fills it: points, pointViews, pointWeights, colors, normals."""
	points: np.ndarray            # (n, 3) float32
	pointViews: list              # per point: ascending image IDs (np.uint32 arrays)
	pointWeights: list            # per point: float32 weights, parallel to pointViews
	colors: object = None         # (n, 3) uint8
	normals: object = None        # (n, 3) float32
	projs: list = None            # per point: (k, 2) uint16 pixel coordinates of its views
	nDepths: int = 0


def FuseDepthMaps(views, nMinViewsFuse: int = 2, fDepthDiffThreshold: float = 0.01, fNormalDiffThreshold: float = 25.0,
		bEstimateColor: bool = True, bEstimateNormal: bool = True) -> PointCloud:
	"""DepthMapsData::FuseDepthMaps (libs/MVS/SceneDensify.cpp:1372-1646).  views[i] (index = image ID): dict with depth (h, w)
	float32 — MODIFIED in place like the reference's depth-maps (depths behind an accepted point are zeroed) — or None, normal
	(h, w, 3) / conf (h, w) / color (h, w, 3) uint8 or None, K R C, neighbors (image IDs, best first) and n_scene_neighbors (the
	connection score).
	numpy maps take b200mvs_fuse_depth_maps (host code: the sequential loop).  CUDA tensors (every map on one device, depth
	contiguous) take b200mvs_fuse_depth_maps_device on a context kept per device: the same point cloud, bit for bit, with the
	pixels of each image resolved in parallel; a neighbour list must not repeat an image ID there."""
	maps = (("depth", "float32", ()), ("normal", "float32", (3,)), ("conf", "float32", ()), ("color", "uint8", (3,)))
	return _cloud_call("FuseDepthMaps", "fuse_depth_maps", views, maps,
		(nMinViewsFuse, fDepthDiffThreshold, fNormalDiffThreshold, bEstimateColor, bEstimateNormal), fuse=True)


def _image_table(where: str, views, device, maps, fuse: bool = False):
	"""the b200mvs_fuse_view table of FuseDepthMaps, MergeDepthMaps and the point-cloud calls -> (table, keepalive).  maps: (key,
	dtype, channels) of the maps the call reads; a map's size is the size of the first map given.  fuse (FuseDepthMaps): depth
	comes first and is modified in place, so it is passed as given and a host depth-map must be writeable; a view without one has
	no other map; and the neighbour fields are set."""
	arr = (_lib.FuseView*len(views))()
	keep = []
	for i, v in enumerate(views):
		o = arr[i]
		size = None
		for key, dt, ch in maps:
			a = v.get(key)
			in_place = fuse and key == "depth"
			if not in_place:
				a = a.contiguous() if _is_torch(a) and a.is_cuda else _host(a, dt, device)
			keep.append(a)
			shape = (None, None)+ch if size is None else size+ch
			setattr(o, key, _arg(where, "views[%d].%s" % (i, key), a, dt, shape, device))
			if in_place and device is None and a is not None and not a.flags.writeable:
				raise ValueError("%s: views[%d].depth must be writeable (it is modified in place)" % (where, i))
			if a is not None and size is None:
				size = tuple(a.shape[:2])
				o.height, o.width = size
			if fuse and size is None:
				break
		for name in ("K", "R", "C"):
			getattr(o, name)[:] = list(np.asarray(v[name], np.float64).ravel())
		if fuse:
			nb = np.ascontiguousarray(v.get("neighbors", []), np.uint32)
			keep.append(nb)
			o.neighbors = nb.ctypes.data if nb.size else None
			o.nNeighbors = int(nb.size)
			o.nSceneNeighbors = int(v.get("n_scene_neighbors", nb.size))
	return arr, keep


def _cloud_call(where: str, name: str, views, maps, params, fuse: bool = False) -> PointCloud:
	"""FuseDepthMaps (fuse) or MergeDepthMaps -> PointCloud: b200mvs_<name> for numpy maps, or b200mvs_<name>_device on the context
	of the device of the first tensor depth-map.  params: the fields of b200mvs_fuse_params."""
	lib = _lib.load()
	first = next((v["depth"] for v in views if _is_torch(v.get("depth"))), None)
	device = None if first is None else _cuda_index(first)
	arr, keep = _image_table(where, views, device, maps, fuse)
	n, md, mn, color, normal = params
	prm = _lib.FuseParams(int(n), float(md), float(mn), int(bool(color)), int(bool(normal)))
	cloud = C.c_void_p()
	if device is not None:
		ctx = _device_context(first.device)
		ctx._call(name + "_device", arr, len(views), C.byref(prm), C.byref(cloud), _stream_handle(ctx.device), C.byref(ctx.stats))
	else:
		rc = getattr(lib, "b200mvs_" + name)(arr, len(views), C.byref(prm), C.byref(cloud))
		if rc:
			raise _lib.B200MVSError("b200mvs_%s failed with status %d (bad view description)" % (name, rc))
	try:
		return _point_cloud(lib, cloud, weights=fuse)
	finally:
		lib.b200mvs_pointcloud_free(cloud)


def _point_cloud(lib, cloud, weights: bool = True) -> PointCloud:
	"""copy a b200mvs_pointcloud into a PointCloud; weights=False: a cloud without weights (MergeDepthMaps), pointWeights None"""
	m = int(lib.b200mvs_pointcloud_size(cloud))
	def take(fn, count, dt):
		p = fn(cloud)
		return np.ctypeslib.as_array(p, shape=(count,)).astype(dt, copy=True) if (count and p) else None
	off = take(lib.b200mvs_pointcloud_view_offsets, m+1, np.uint32)
	total = int(off[-1]) if off is not None else 0
	pts = take(lib.b200mvs_pointcloud_points, 3*m, np.float32)
	vs = take(lib.b200mvs_pointcloud_views, total, np.uint32); ws = take(lib.b200mvs_pointcloud_weights, total, np.float32)
	pj = take(lib.b200mvs_pointcloud_projs, 2*total, np.uint16)
	nr = take(lib.b200mvs_pointcloud_normals, 3*m, np.float32); cl = take(lib.b200mvs_pointcloud_colors, 3*m, np.uint8)
	return PointCloud(points=pts.reshape(-1, 3) if pts is not None else np.zeros((0, 3), np.float32),
		pointViews=[vs[off[i]:off[i+1]] for i in range(m)], pointWeights=[ws[off[i]:off[i+1]] for i in range(m)] if weights else None,
		colors=None if cl is None else cl.reshape(-1, 3), normals=None if nr is None else nr.reshape(-1, 3),
		projs=[pj[2*off[i]:2*off[i+1]].reshape(-1, 2) for i in range(m)], nDepths=int(lib.b200mvs_pointcloud_depths(cloud)))


def FuseRoundStats():
	"""What each round (image) of the last device FuseDepthMaps call on each device did: {device index: list of dicts with image,
	iterations (of the acceptance fixed point), candidates, edges (claim and zero), shared (edges whose neighbour pixel another
	candidate also reaches) and ms (device time)}."""
	out = {}
	for index, ctx in _DEVICE_CTX.items():
		n = C.c_int()
		ctx._call("fuse_round_stats", 0, C.byref(n), None, None, None, None, None, None)
		m = n.value
		img, it = np.zeros(m, np.int32), np.zeros(m, np.int32)
		cand, edges, shared, ms = np.zeros(m, np.uint64), np.zeros(m, np.uint64), np.zeros(m, np.uint64), np.zeros(m, np.float32)
		ctx._call("fuse_round_stats", m, C.byref(n), img.ctypes.data_as(C.POINTER(C.c_int)), it.ctypes.data_as(C.POINTER(C.c_int)),
			cand.ctypes.data, edges.ctypes.data, shared.ctypes.data, ms.ctypes.data)
		out[index] = [dict(image=int(img[i]), iterations=int(it[i]), candidates=int(cand[i]), edges=int(edges[i]), shared=int(shared[i]),
			ms=float(ms[i])) for i in range(m)]
	return out



# The point-cloud calls after the fusion live in point_cloud.py, which builds on this module; they are re-exported here on first
# use, so that either module can be imported first.
_POINT_CLOUD_CALLS = ("MergeDepthMaps", "EstimatePointColors", "EstimatePointNormals", "PointKNN", "PointCloudVisibility",
	"PointCloudFilter")


def __getattr__(name):
	if name in _POINT_CLOUD_CALLS:
		from . import point_cloud
		return getattr(point_cloud, name)
	raise AttributeError("module %r has no attribute %r" % (__name__, name))
