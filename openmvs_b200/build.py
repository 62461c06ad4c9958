"""In-tree build of the C-ABI shared library (nvcc, sm_90a only; no JIT cache)."""
from __future__ import annotations

import glob
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB_PATH = os.path.join(HERE, "libb200mvs.so")
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
	"-Xcompiler", "-fPIC", "-shared", "-Xlinker", "--no-undefined"]


def sources():
	return sorted(glob.glob(os.path.join(HERE, "csrc", "*.cu")))


def is_stale() -> bool:
	if not os.path.exists(LIB_PATH):
		return True
	t = os.path.getmtime(LIB_PATH)
	deps = sources() + glob.glob(os.path.join(HERE, "csrc", "*.cuh")) + glob.glob(os.path.join(HERE, "csrc", "*.h")) + \
		glob.glob(os.path.join(ROOT, "include", "*.h"))
	return any(os.path.getmtime(d) > t for d in deps)


def build_extension(force: bool = False, verbose: bool = False) -> str:
	"""Compile openmvs_b200/csrc/*.cu into openmvs_b200/libb200mvs.so for sm_90a."""
	if not force and not is_stale():
		return LIB_PATH
	nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
	if not os.path.exists(nvcc):
		raise RuntimeError("nvcc not found and %s is missing or stale" % LIB_PATH)
	# build to a temporary name under a file lock and rename: concurrent ranks (torchrun) never see a half-written library
	import fcntl
	with open(LIB_PATH+".lock", "w") as lock:
		fcntl.flock(lock, fcntl.LOCK_EX)
		if not force and not is_stale():
			return LIB_PATH
		tmp = "%s.tmp.%d" % (LIB_PATH, os.getpid())
		cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", tmp] + sources()
		try:
			subprocess.check_call(cmd, cwd=ROOT)
			os.replace(tmp, LIB_PATH)
		finally:
			if os.path.exists(tmp):
				os.unlink(tmp)
	return LIB_PATH


if __name__ == "__main__":
	print(build_extension(force=True, verbose=True))
