""".dmap depth-data files — the wire format either side of the hot path (SURVEY.md §8(f) rank 1).

ExportDepthDataRaw / ImportDepthDataRaw follow the reference's raw layout
(libs/MVS/DepthMap.cpp:1874-2037, header `HeaderDepthDataRaw` libs/MVS/Interface.h:773-792):

  u16 'DR' | u8 type (HAS_DEPTH=1, HAS_NORMAL=2, HAS_CONF=4, HAS_VIEWS=8) | u8 padding
  u32 imageWidth, imageHeight | u32 depthWidth, depthHeight | f32 dMin, dMax
  u16 nFileNameSize, chars | u32 nIDs, u32 IDs[nIDs] (reference view first)
  f64 K[9], R[9], C[3] | f32 depth[h][w] | f32 normal[h][w][3] | f32 conf[h][w] | u8 views[h][w][4]

Host-side plumbing (numpy); files are written atomically (.tmp + rename) like DepthData::Save
(libs/MVS/DepthMap.cpp:237-251).

The .dimap disparity-data files of the SGM path (ExportDisparityDataRaw[Full] / ImportDisparityDataRaw[Full]) are the hand-off
between SGM matching (fusion-mode -1) and the fusion of the pairs into depth-maps (fusion-mode -2).
"""
from __future__ import annotations

import os
import struct

import numpy as np

HAS_DEPTH, HAS_NORMAL, HAS_CONF, HAS_VIEWS = 1, 2, 4, 8


def ExportDepthDataRaw(fileName, imageFileName, IDs, imageSize, K, R, C, dMin, dMax, depthMap, normalMap=None, confMap=None, viewsMap=None) -> bool:
	depth = np.ascontiguousarray(depthMap, np.float32)
	h, w = depth.shape
	if not (1 < len(IDs) < 256) or w > imageSize[0] or h > imageSize[1]:
		raise ValueError("IDs must hold the reference and at least one neighbour; the depth-map may not exceed the image")
	typ = HAS_DEPTH
	blobs = [depth.tobytes()]
	for arr, flag, shape, dt in ((normalMap, HAS_NORMAL, (h, w, 3), np.float32), (confMap, HAS_CONF, (h, w), np.float32), (viewsMap, HAS_VIEWS, (h, w, 4), np.uint8)):
		if arr is not None:
			a = np.ascontiguousarray(arr, dt)
			if a.shape != shape:
				raise ValueError("map shape %s, expected %s" % (a.shape, shape))
			typ |= flag
			blobs.append(a.tobytes())
	name = os.path.relpath(os.path.abspath(imageFileName), os.path.dirname(os.path.abspath(fileName))).encode()
	tmp = fileName+".tmp"
	with open(tmp, "wb") as f:
		f.write(b"DR"+struct.pack("<BBIIIIff", typ, 0, imageSize[0], imageSize[1], w, h, float(dMin), float(dMax)))
		f.write(struct.pack("<H", len(name))+name)
		f.write(struct.pack("<I", len(IDs))+np.asarray(IDs, np.uint32).tobytes())
		f.write(np.asarray(K, np.float64).reshape(9).tobytes()+np.asarray(R, np.float64).reshape(9).tobytes()+np.asarray(C, np.float64).reshape(3).tobytes())
		for b in blobs:
			f.write(b)
	os.replace(tmp, fileName)
	return True


def ImportDepthDataRaw(fileName, flags: int = 15) -> dict:
	"""-> dict(imageFileName, IDs, imageSize, K, R, C, dMin, dMax, depthMap, normalMap, confMap, viewsMap);
	flags selects which optional maps to return (HAS_* bits), like the reference's `flags` argument."""
	with open(fileName, "rb") as f:
		head = f.read(28)
		if len(head) != 28 or head[:2] != b"DR":
			raise ValueError("%s is not a depth-data file" % fileName)
		typ, _, iw, ih, w, h, dmin, dmax = struct.unpack("<BBIIIIff", head[2:])
		if not (typ & HAS_DEPTH) or w == 0 or h == 0 or iw < w or ih < h:
			raise ValueError("invalid depth-data header")
		n, = struct.unpack("<H", f.read(2))
		name = f.read(n).decode()
		nids, = struct.unpack("<I", f.read(4))
		ids = np.frombuffer(f.read(4*nids), np.uint32).copy()
		K = np.frombuffer(f.read(72), np.float64).reshape(3, 3).copy()
		R = np.frombuffer(f.read(72), np.float64).reshape(3, 3).copy()
		Cc = np.frombuffer(f.read(24), np.float64).copy()
		out = dict(imageFileName=name, IDs=ids, imageSize=(iw, ih), K=K, R=R, C=Cc, dMin=dmin, dMax=dmax,
			normalMap=None, confMap=None, viewsMap=None)
		out["depthMap"] = np.frombuffer(f.read(4*w*h), np.float32).reshape(h, w).copy()
		for key, flag, count, dt, shape in (("normalMap", HAS_NORMAL, 12*w*h, np.float32, (h, w, 3)), ("confMap", HAS_CONF, 4*w*h, np.float32, (h, w)), ("viewsMap", HAS_VIEWS, 4*w*h, np.uint8, (h, w, 4))):
			if typ & flag:
				raw = f.read(count)
				if flags & flag:
					out[key] = np.frombuffer(raw, dt).reshape(shape).copy()
	return out


NO_DISP = 32767          # SemiGlobalMatcher::NO_DISP
NO_ACCUMCOST = 65535     # SemiGlobalMatcher::NO_ACCUMCOST
_DIMAP_HEAD = struct.Struct("<ii9d16dhii")   # image size, H, Q, subpixelSteps, map columns and rows (packed, no padding)


def ExportDisparityDataRaw(fileName, disparityMap, costMap, imageSize, H, Q, subpixelSteps) -> bool:
	""".dimap file of one SGM pair (SemiGlobalMatcher::ExportDisparityDataRaw, libs/MVS/SemiGlobalMatcher.cpp:2094-2122), packed little
	endian: int32 image width and height, 9 doubles H, 16 doubles Q, int16 subpixelSteps, int32 columns and rows of the map, the int16
	disparity map (disparity * subpixelSteps, NO_DISP where invalid), then the uint16 cost map when there is one."""
	disp = np.ascontiguousarray(disparityMap, "<i2")
	rows, cols = disp.shape
	cost = None if costMap is None else np.ascontiguousarray(costMap, "<u2")
	if cost is not None and cost.shape != disp.shape:
		raise ValueError("cost map of shape %s for a disparity map of shape %s" % (cost.shape, disp.shape))
	head = _DIMAP_HEAD.pack(int(imageSize[0]), int(imageSize[1]), *np.asarray(H, np.float64).reshape(9).tolist(),
		*np.asarray(Q, np.float64).reshape(16).tolist(), int(subpixelSteps), cols, rows)
	with open(fileName, "wb") as f:
		f.write(head)
		f.write(disp.tobytes())
		if cost is not None:
			f.write(cost.tobytes())
	return True


def ExportDisparityDataRawFull(fileName, disparityMap, costMap, imageSize, H, Q, subpixelSteps) -> bool:
	"""ExportDisparityDataRaw of the maps padded with the 3-pixel border the matcher leaves out (NO_DISP / NO_ACCUMCOST;
	SemiGlobalMatcher.cpp:2124-2138): the form SGM matching writes and fusion reads."""
	disp = np.asarray(disparityMap)
	pad = lambda m, v: np.pad(np.asarray(m), 3, constant_values=v)
	return ExportDisparityDataRaw(fileName, pad(disp, NO_DISP), None if costMap is None else pad(costMap, NO_ACCUMCOST), imageSize, H, Q,
		subpixelSteps)


def ImportDisparityDataRaw(fileName) -> dict:
	"""-> dict(disparityMap (int16), costMap (uint16 or None: no bytes after the disparity map), imageSize, H (3x3), Q (4x4),
	subpixelSteps) of a .dimap file (SemiGlobalMatcher::ImportDisparityDataRaw, SemiGlobalMatcher.cpp:2140-2172)"""
	with open(fileName, "rb") as f:
		raw = f.read()
	if len(raw) < _DIMAP_HEAD.size:
		raise ValueError("%s is too short for a disparity-data file" % fileName)
	v = _DIMAP_HEAD.unpack_from(raw)
	iw, ih, H, Q, steps, cols, rows = v[0], v[1], v[2:11], v[11:27], v[27], v[28], v[29]
	if iw <= 0 or ih <= 0 or cols <= 0 or rows <= 0:
		raise ValueError("invalid disparity-data header")
	n = cols*rows
	rest = raw[_DIMAP_HEAD.size:]
	if len(rest) not in (2*n, 4*n):
		raise ValueError("%s holds %d bytes of maps, expected %d or %d" % (fileName, len(rest), 2*n, 4*n))
	disp = np.frombuffer(rest[:2*n], "<i2").reshape(rows, cols).astype(np.int16)
	cost = np.frombuffer(rest[2*n:], "<u2").reshape(rows, cols).astype(np.uint16) if len(rest) == 4*n else None
	return dict(disparityMap=disp, costMap=cost, imageSize=(iw, ih), H=np.array(H, np.float64).reshape(3, 3),
		Q=np.array(Q, np.float64).reshape(4, 4), subpixelSteps=int(steps))


def ImportDisparityDataRawFull(fileName) -> dict:
	"""ImportDisparityDataRaw with the 3-pixel border cropped (SemiGlobalMatcher.cpp:2174-2184): the maps of the valid region"""
	d = ImportDisparityDataRaw(fileName)
	crop = lambda m: None if m is None else np.ascontiguousarray(m[3:-3, 3:-3])
	if min(d["disparityMap"].shape) <= 6:
		raise ValueError("a full disparity map must be larger than its 3-pixel border")
	d["disparityMap"], d["costMap"] = crop(d["disparityMap"]), crop(d["costMap"])
	return d


class AsyncDepthDataWriter:
	"""Asynchronous emission of `.dmap` files (SURVEY.md §8(f) rank 1, second half).

	The reference saves a depth-map from its event loop after the estimation of the next image has been queued
	(EVT_SAVEDEPTHMAP, libs/MVS/SceneDensify.cpp:2065,2092-2113; DepthData::Save libs/MVS/DepthMap.cpp:237-251), so the disk
	write overlaps the next estimation.  Here `submit()` returns at once: device-resident maps (torch CUDA tensors) are copied to
	pinned host buffers on a side stream that waits for the producing stream, and a worker thread writes the file when the copy
	has landed; host arrays go straight to the worker.  `flush()` waits for everything submitted and re-raises the first error.
	At most `max_pending` files are in flight (their pinned buffers are recycled), so a slow disk throttles the caller instead of
	growing memory without bound."""

	def __init__(self, max_pending: int = 4):
		import queue, threading
		self._q = queue.Queue()
		self._slots = threading.Semaphore(max_pending)
		self._errors = []
		self._pool = {}          # (shape, dtype) -> list of free pinned tensors
		self._lock = threading.Lock()
		self._stream = None
		self._thread = threading.Thread(target=self._run, name="dmap-writer", daemon=True)
		self._thread.start()
		self.files_written = 0

	def _pinned(self, t):
		import torch
		key = (tuple(t.shape), t.dtype)
		with self._lock:
			free = self._pool.setdefault(key, [])
			if free:
				return free.pop()
		return torch.empty(t.shape, dtype=t.dtype, pin_memory=True)

	def _release(self, bufs):
		with self._lock:
			for b in bufs:
				self._pool.setdefault((tuple(b.shape), b.dtype), []).append(b)

	def submit(self, fileName, imageFileName, IDs, imageSize, K, R, C, dMin, dMax, depthMap, normalMap=None, confMap=None, viewsMap=None):
		"""Queue one file; the maps may be numpy arrays or torch tensors (CUDA tensors are read in the current stream's order:
		work queued on it before this call is finished before the copy starts, work queued after it waits for the copy)."""
		# host arrays are snapshotted here, device maps by the ordered copy below: the caller may reuse both right away
		maps = [m if (m is None or hasattr(m, "is_cuda")) else np.array(m, copy=True) for m in (depthMap, normalMap, confMap, viewsMap)]
		self._slots.acquire()
		event, bufs = None, []
		try:
			import torch
			cuda = [m for m in maps if m is not None and hasattr(m, "is_cuda") and m.is_cuda]
			if cuda:
				dev = cuda[0].device
				if self._stream is None or self._stream.device != dev:
					self._stream = torch.cuda.Stream(device=dev)
				self._stream.wait_stream(torch.cuda.current_stream(dev))
				with torch.cuda.stream(self._stream):
					for i, m in enumerate(maps):
						if m is not None and hasattr(m, "is_cuda") and m.is_cuda:
							m = m.contiguous()
							m.record_stream(self._stream)
							b = self._pinned(m)
							b.copy_(m, non_blocking=True)
							bufs.append(b); maps[i] = b
					event = torch.cuda.Event()
					event.record(self._stream)
				# later work on the producing stream must not overwrite the maps before the copy has read them
				torch.cuda.current_stream(dev).wait_event(event)
		except ImportError:
			pass
		self._q.put((fileName, imageFileName, list(IDs), tuple(imageSize), np.array(K, np.float64), np.array(R, np.float64), np.array(C, np.float64),
			float(dMin), float(dMax), maps, event, bufs))

	def _run(self):
		while True:
			job = self._q.get()
			if job is None:
				self._q.task_done()
				return
			fileName, imageFileName, IDs, imageSize, K, R, C, dMin, dMax, maps, event, bufs = job
			try:
				if event is not None:
					event.synchronize()
				host = [None if m is None else (m.numpy() if hasattr(m, "numpy") else np.asarray(m)) for m in maps]
				ExportDepthDataRaw(fileName, imageFileName, IDs, imageSize, K, R, C, dMin, dMax, host[0], host[1], host[2], host[3])
				self.files_written += 1
			except Exception as e:   # reported by flush()
				self._errors.append((fileName, e))
			finally:
				self._release(bufs)
				self._slots.release()
				self._q.task_done()

	def flush(self):
		self._q.join()
		if self._errors:
			name, e = self._errors[0]
			self._errors = []
			raise RuntimeError("writing %s failed: %r" % (name, e))

	def close(self):
		self._q.join()
		self._q.put(None)
		self._thread.join()
		if self._errors:
			name, e = self._errors[0]
			raise RuntimeError("writing %s failed: %r" % (name, e))

	def __enter__(self):
		return self

	def __exit__(self, *exc):
		self.close()
		return False
