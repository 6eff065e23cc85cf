#!/bin/bash
# Host-side memory / UB check of the shim without a GPU: cusparse_shim.cpp + config.cpp + real_cusparse.cpp compiled with
# -fsanitize=address,undefined, linked with the library's ordinary CUDA objects (cudalibrarysamples_b200/build/*.cu.o, built by
# __graft_entry__.build()), then the descriptor / routing script of tests/test_descriptors_cpu.py is run against that build.
# Round 2: clean ("OK", no sanitizer report).
set -e
cd "$(dirname "$0")/../cudalibrarysamples_b200"
mkdir -p build/asan
for f in cusparse_shim config real_cusparse; do
  g++ -O1 -g -std=c++17 -fPIC -fsanitize=address,undefined -fno-omit-frame-pointer -w -I/usr/local/cuda/include -c csrc/$f.cpp -o build/asan/$f.o
done
g++ -shared -fsanitize=address,undefined -o build/asan/libb200spmv_asan.so build/asan/cusparse_shim.o build/asan/config.o \
    build/asan/real_cusparse.o build/*.cu.o \
    -L/usr/local/cuda/lib64 -lcudart -ldl -lpthread
cd ..
python - <<'PY'
import os, re, subprocess, sys, textwrap
src = open("tests/test_descriptors_cpu.py").read()
script = textwrap.dedent(re.search(r'SCRIPT = textwrap.dedent\("""(.*?)"""\)', src, re.S).group(1))
real = "/usr/local/cuda/lib64/libcusparse.so.12"
env = dict(os.environ, B200SPMV_CUSPARSE=real, ASAN_OPTIONS="detect_leaks=0:protect_shadow_gap=0",
           LD_PRELOAD=subprocess.check_output(["gcc", "-print-file-name=libasan.so"], text=True).strip())
p = subprocess.run([sys.executable, "-c", script, "cudalibrarysamples_b200/build/asan/libb200spmv_asan.so", real], capture_output=True, text=True, env=env)
print(p.stdout.strip()[-100:])
bad = [l for l in p.stderr.splitlines() if "Sanitizer" in l or "runtime error" in l]
print("sanitizer reports:", bad if bad else "none")
sys.exit(p.returncode or (1 if bad else 0))
PY
