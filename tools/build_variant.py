#!/usr/bin/env python
"""A/B builds of the product library: recompiles the named kernel translation units with extra nvcc flags and links them with the
other (unchanged) objects into raytracingdenoiser_b200/libnrd_b200_<name>.so.  Select it at run time with
NRD_B200_LIB=<path> (raytracingdenoiser_b200/nrd.py).   python tools/build_variant.py ta4 reblur_temporal.cu -DNRD_B200_TA_MIN_BLOCKS=4"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from raytracingdenoiser_b200 import build as b  # noqa: E402

name, unit = sys.argv[1], sys.argv[2]
extra = sys.argv[3:]
b.build_product()
objs = []
for f in sorted(os.listdir(b.OBJ)):
    if f.endswith(".o"):
        objs.append(os.path.join(b.OBJ, f))
vdir = os.path.join(b.OBJ, "variant_" + name)
os.makedirs(vdir, exist_ok=True)
src = os.path.join(b.CSRC, "device", unit)
base = unit.replace(".", "_")
for suffix, flags in (("", []), ("_single", ["-DNRD_B200_NO_STRIPS"])):
    obj = os.path.join(vdir, base + suffix + ".o")
    cmd = [b.NVCC] + b.NVCC_FLAGS + flags + extra + ["-c", src, "-o", obj]
    subprocess.run(cmd, check=True)
    objs = [o for o in objs if os.path.basename(o) != base + suffix + ".o"] + [obj]
lib = os.path.join(b.PKG, "libnrd_b200_%s.so" % name)
subprocess.run([b.NVCC, "-shared", "-o", lib] + objs + b.ARCH + ["-Xcompiler", "-fPIC", "-lcudart_static", "-ldl", "-lrt", "-lpthread"], check=True)
print(lib)
