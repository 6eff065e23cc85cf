#!/usr/bin/env python
"""Parameter sweeps for the CSR tile kernel.

  python scripts/sweep.py build            (CPU container)  nvcc-build one .so per variant into build/variants/
  python scripts/sweep.py run [workloads]  (GPU box)        time every variant + the closed library on each workload

Variants are -D overrides of the tunables at the top of csrc/spmv_csr.cu.
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
VDIR = os.path.join(ROOT, "cudalibrarysamples_b200", "build", "variants")

VARIANTS = {
    # tag: dict(TILE, LONG, BLOCK, BATCH, MIN_CTAS)
    "t2048_b256_k4": dict(TILE=2048, LONG=512, BLOCK=256, BATCH=4, MIN=1),
    "t2048_b256_k4_occ6": dict(TILE=2048, LONG=512, BLOCK=256, BATCH=4, MIN=6),
    "t2048_b256_k4_occ8": dict(TILE=2048, LONG=512, BLOCK=256, BATCH=4, MIN=8),
    "t2048_b256_k4_occ5": dict(TILE=2048, LONG=512, BLOCK=256, BATCH=4, MIN=5),
    "t2048_b256_k2_occ8": dict(TILE=2048, LONG=512, BLOCK=256, BATCH=2, MIN=8),
    "t2048_b256_k8": dict(TILE=2048, LONG=512, BLOCK=256, BATCH=8, MIN=1),
    "t2048_b128_k4": dict(TILE=2048, LONG=512, BLOCK=128, BATCH=4, MIN=1),
    "t2048_b128_k8": dict(TILE=2048, LONG=512, BLOCK=128, BATCH=8, MIN=1),
    "t1024_b128_k4": dict(TILE=1024, LONG=256, BLOCK=128, BATCH=4, MIN=1),
    "t1024_b256_k4": dict(TILE=1024, LONG=256, BLOCK=256, BATCH=4, MIN=1),
    "t4096_b256_k8": dict(TILE=4096, LONG=1024, BLOCK=256, BATCH=8, MIN=1),
    "t4096_b512_k4": dict(TILE=4096, LONG=1024, BLOCK=512, BATCH=4, MIN=1),
    "t3072_b256_k4": dict(TILE=3072, LONG=512, BLOCK=256, BATCH=4, MIN=1),
}


ABL = {f"abl{a}_occ6": dict(TILE=2048, LONG=512, BLOCK=256, BATCH=4, MIN=6, ABL=a) for a in (1, 2, 3)}
if os.environ.get("SWEEP_SET") == "occ":
    VARIANTS = {f"t2048_b256_k{k}_occ{o}": dict(TILE=2048, LONG=512, BLOCK=256, BATCH=k, MIN=o) for k in (4, 8) for o in (4, 5, 6, 7)}
    VARIANTS.update({f"t1024_b128_k{k}_occ{o}": dict(TILE=1024, LONG=256, BLOCK=128, BATCH=k, MIN=o) for k in (4, 8) for o in (8, 12)})
    VARIANTS.update({f"t1024_b256_k4_occ{o}": dict(TILE=1024, LONG=256, BLOCK=256, BATCH=4, MIN=o) for o in (6, 8)})
if os.environ.get("SWEEP_SET") == "pipe":
    VARIANTS = {f"pipe_t2048_b256_o{po}_occ{o}": dict(TILE=2048, LONG=512, BLOCK=256, BATCH=4, MIN=o, KERNEL=1, OFFS=po)
                for po in (2, 4) for o in (3, 4, 5, 6)}
    VARIANTS.update({f"pipe_t1024_b128_o{po}_occ{o}": dict(TILE=1024, LONG=256, BLOCK=128, BATCH=4, MIN=o, KERNEL=1, OFFS=po)
                     for po in (4,) for o in (6, 8, 10, 12)})
    VARIANTS.update({f"pipe_t1024_b256_o2_occ{o}": dict(TILE=1024, LONG=256, BLOCK=256, BATCH=4, MIN=o, KERNEL=1, OFFS=2)
                     for o in (4, 6, 8)})
    VARIANTS.update({f"tile_t1024_b128_k8_occ12": dict(TILE=1024, LONG=256, BLOCK=128, BATCH=8, MIN=12, KERNEL=0)})
if os.environ.get("SWEEP_SET") == "red":
    VARIANTS = {}
    for rr, ru in ((4, 2), (2, 4), (4, 1), (2, 2)):
        for o in (3, 4, 5):
            VARIANTS[f"pipe_r{rr}u{ru}_occ{o}"] = dict(TILE=2048, LONG=512, BLOCK=256, BATCH=4, MIN=o, KERNEL=1, OFFS=4, RR=rr, RU=ru)
        VARIANTS[f"tile_r{rr}u{ru}_occ5"] = dict(TILE=2048, LONG=512, BLOCK=256, BATCH=4, MIN=5, KERNEL=0, RR=rr, RU=ru)
        VARIANTS[f"pipe1024_r{rr}u{ru}_occ8"] = dict(TILE=1024, LONG=256, BLOCK=128, BATCH=4, MIN=8, KERNEL=1, OFFS=4, RR=rr, RU=ru)
if os.environ.get("SWEEP_SET") == "ws":
    VARIANTS = {}
    #            tile  long gw rw rg st un ctas
    for cfg in [(2048, 512, 8, 4, 2, 4, 8, 1), (2048, 512, 4, 4, 1, 2, 8, 2), (2048, 512, 4, 4, 1, 3, 8, 2),
                (1024, 256, 4, 4, 1, 3, 8, 3), (1024, 256, 4, 4, 1, 3, 8, 4), (1024, 256, 4, 2, 1, 3, 8, 4),
                (1024, 256, 2, 2, 1, 3, 8, 6), (1024, 256, 4, 2, 1, 2, 8, 5), (512, 128, 2, 2, 1, 3, 8, 8),
                (1024, 256, 4, 4, 1, 4, 8, 3)]:
        t, l, gw, rw, rg, st, un, ct = cfg
        VARIANTS[f"ws_t{t}_g{gw}_r{rw}x{rg}_s{st}_c{ct}"] = dict(TILE=t, LONG=l, BLOCK=256, BATCH=4, MIN=4, WS=cfg[2:])
if os.environ.get("SWEEP_SET") == "small":
    VARIANTS = {}
    for (t, l, bl, k, o) in [(512, 128, 128, 6, 16), (512, 128, 128, 3, 16), (512, 128, 128, 6, 12), (768, 256, 128, 9, 12),
                             (1024, 256, 128, 11, 12), (1024, 256, 128, 4, 12), (512, 128, 64, 11, 24), (256, 64, 64, 6, 32),
                             (1024, 256, 256, 6, 6), (2048, 512, 256, 4, 5), (384, 128, 128, 5, 16), (640, 128, 128, 7, 14)]:
        VARIANTS[f"tile_t{t}_l{l}_b{bl}_k{k}_occ{o}"] = dict(TILE=t, LONG=l, BLOCK=bl, BATCH=k, MIN=o, KERNEL=0)
if os.environ.get("SWEEP_SET") == "rw":
    VARIANTS = {}
    for (t, l, bl, o, rr, ru) in [(2048, 512, 256, 4, 4, 2), (2048, 512, 256, 6, 2, 2), (2048, 512, 256, 5, 4, 1), (2048, 512, 256, 8, 2, 1),
                                  (1024, 256, 128, 8, 4, 2), (1024, 256, 128, 12, 2, 2), (1024, 256, 256, 6, 2, 2), (4096, 1024, 256, 4, 4, 2),
                                  (2048, 512, 256, 4, 2, 4), (2048, 512, 128, 8, 4, 2), (512, 128, 128, 12, 2, 2), (2048, 512, 256, 3, 4, 4)]:
        VARIANTS[f"rw_t{t}_b{bl}_occ{o}_r{rr}u{ru}"] = dict(TILE=t, LONG=l, BLOCK=bl, BATCH=4, MIN=o, KERNEL=3, RW=(rr, ru))
if os.environ.get("SWEEP_SET") == "final":
    VARIANTS = {
        "tile_occ5": dict(TILE=2048, LONG=512, BLOCK=256, BATCH=4, MIN=5, KERNEL=0, RR=2, RU=2),
        "tile_occ6": dict(TILE=2048, LONG=512, BLOCK=256, BATCH=4, MIN=6, KERNEL=0, RR=2, RU=2),
        "pipe_occ3": dict(TILE=2048, LONG=512, BLOCK=256, BATCH=4, MIN=3, KERNEL=1, OFFS=4, RR=2, RU=2),
        "pipe_occ4": dict(TILE=2048, LONG=512, BLOCK=256, BATCH=4, MIN=4, KERNEL=1, OFFS=4, RR=2, RU=4),
        "rw_b128_occ8": dict(TILE=2048, LONG=512, BLOCK=128, BATCH=4, MIN=8, KERNEL=3, RW=(4, 2)),
    }
if os.environ.get("SWEEP_SET") == "ab":
    VARIANTS = {k: {} for k in ['t2048_l256', 't1536_l512_occ6', 't1536_l256_occ6', 't2560_l512_occ4', 't1024_l256_b128_occ10', 't3072_l512_b384_occ3']}
if os.environ.get("SWEEP_SET") == "seg":
    # csr_seg_kernel: tile size, resident CTAs (register cap), batch depth, with / without the staged-product fallback
    VARIANTS = {}
    for (o, k, staged) in [(4, 4, 1), (5, 4, 1), (6, 4, 1), (5, 2, 1), (6, 2, 1), (6, 4, 0), (8, 2, 0), (5, 4, 0), (4, 4, 0), (6, 2, 0)]:
        VARIANTS[f"seg_occ{o}_k{k}_st{staged}"] = dict(SEG=(o, k, staged))
    for (o, k, staged) in [(5, 4, 1), (6, 2, 1), (8, 2, 1), (6, 4, 0), (6, 2, 0), (8, 2, 0), (8, 4, 0)]:
        VARIANTS[f"seg_t1024_b256_occ{o}_k{k}_st{staged}"] = dict(SEG=(o, k, staged), TILE=1024, LONG=256, BLOCK=256)
    VARIANTS["seg_t1024_b128_occ10_k4_st0"] = dict(SEG=(10, 4, 0), TILE=1024, LONG=256, BLOCK=128)
    VARIANTS["seg_t1024_b128_occ12_k4_st1"] = dict(SEG=(12, 4, 1), TILE=1024, LONG=256, BLOCK=128)
    VARIANTS["seg_t512_b128_occ12_k2_st0"] = dict(SEG=(12, 2, 0), TILE=512, LONG=128, BLOCK=128)
    VARIANTS["seg_t3072_b384_occ4_k4_st0"] = dict(SEG=(4, 4, 0), TILE=3072, LONG=512, BLOCK=384)
if os.environ.get("SWEEP_SET") == "flat":
    # csr_flat_kernel: (resident CTAs, batch, warps per CTA, steps per warp chunk, nzrow prefetch)
    VARIANTS = {f"flat_occ{o}_k{k}_w{w}_s{st}_nz{nz}": dict(FLAT=(o, k, w, st, nz)) for (o, k, w, st, nz) in
                [(10, 4, 4, 8, 0), (10, 4, 4, 8, 1), (12, 4, 4, 8, 1), (8, 4, 4, 8, 1), (10, 2, 4, 8, 1),
                 (10, 4, 4, 16, 1), (12, 4, 4, 16, 1), (8, 4, 4, 16, 1), (20, 4, 2, 16, 1), (10, 4, 2, 32, 1), (20, 4, 2, 32, 1),
                 (5, 4, 8, 8, 1), (20, 4, 2, 8, 1), (40, 4, 1, 16, 1), (40, 4, 1, 8, 1)]}
if os.environ.get("SWEEP_SET") == "flat3":
    # csr_flat_kernel: (quiet-step ballot, empty rows scaled by tail CTAs of the main grid)
    VARIANTS = {f"flat3_qb{qb}_et{et}": dict(FLAT3=(qb, et)) for (qb, et) in [(1, 1), (0, 1), (1, 0), (0, 0)]}
if os.environ.get("SWEEP_SET") == "flat4":
    # csr_flat_kernel: deeper load batches / more resident CTAs (the fp32 kernel has registers to spare)
    VARIANTS = {f"flat4_occ{o}_k{k}_w{w}_s{st}": dict(FLAT=(o, k, w, st)) for (o, k, w, st) in
                [(10, 8, 4, 8), (12, 8, 4, 8), (12, 4, 4, 8), (8, 8, 4, 8)]}
if os.environ.get("SWEEP_SET") == "flat_hot":
    # csr_flat_kernel: byte budget of the packed hot columns of x (0 = no hot plan)
    VARIANTS = {f"flat_hot{kb}k": dict(FLATHOT=kb) for kb in (0, 64, 96, 128, 160)}
if os.environ.get("SWEEP_SET") == "flat_l1":
    # csr_flat_kernel: (B200_FLAT_COLD = L1 policy of the cold x gathers, hot budget in KB); run with SWEEP_ROUNDS=3
    VARIANTS = {f"flat_l1_p{p}_h{kb}k": dict(FLATL1=(p, kb)) for p in (0, 1, 2) for kb in (0, 64, 96, 128, 160, 192)}
if os.environ.get("SWEEP_SET") == "short":
    # csr_short_kernel: (warps per CTA, load steps per pass, resident CTAs)
    VARIANTS = {f"short_w{w}_s{st}_occ{o}": dict(SHORT=(w, st, o)) for (w, st, o) in
                [(8, 8, 5), (8, 8, 4), (8, 8, 6), (4, 8, 10), (4, 8, 8), (8, 6, 6), (8, 6, 8), (16, 8, 2), (8, 12, 4), (8, 16, 3)]}
if os.environ.get("SWEEP_SET") == "ablate":
    VARIANTS = dict(ABL, t2048_b256_k4_occ6=VARIANTS["t2048_b256_k4_occ6"])


def flags(v):
    if "FLAT" in v:
        o, k, w, st = v["FLAT"][:4]
        return [f"-DB200_FLAT_MIN_CTAS={o}", f"-DB200_FLAT_BATCH={k}", f"-DB200_FLAT_WARPS={w}", f"-DB200_FLAT_STEPS={st}"]
    if "FLAT3" in v:
        return [f"-DB200_FLAT_QUIET_BALLOT={v['FLAT3'][0]}", f"-DB200_FLAT_EMPTY_TAIL={v['FLAT3'][1]}"]
    if "FLATHOT" in v:
        return [f"-DB200_FLAT_HOT_BYTES={v['FLATHOT'] * 1024}"]
    if "FLATL1" in v:
        p, kb = v["FLATL1"]
        return [f"-DB200_FLAT_COLD={p}", f"-DB200_FLAT_HOT_BYTES={kb * 1024}"]
    if "SHORT" in v:
        w, st, o = v["SHORT"]
        return [f"-DB200_SHORT_WARPS={w}", f"-DB200_SHORT_STEPS={st}", f"-DB200_SHORT_MIN_CTAS={o}"]
    if "SEG" in v:
        o, k, staged = v["SEG"]
        base = dict(TILE=v.get("TILE", 2048), LONG=v.get("LONG", 512), BLOCK=v.get("BLOCK", 256), BATCH=4, MIN=5)
        return flags(base) + ["-DB200_CSR_KERNEL=5", f"-DB200_SEG_MIN_CTAS={o}", f"-DB200_SEG_BATCH={k}", f"-DB200_SEG_STAGED={staged}"]
    if "ABL" in v:
        return flags({k: x for k, x in v.items() if k != "ABL"}) + [f"-DB200_CSR_ABLATE={v['ABL']}"]
    if "RW" in v:
        return flags({k: x for k, x in v.items() if k != "RW"}) + [f"-DB200_RW_ROWS={v['RW'][0]}", f"-DB200_RW_U={v['RW'][1]}"]
    if "WS" in v:
        gw, rw, rg, st, un, ct = v["WS"]
        return flags({k: x for k, x in v.items() if k != "WS"}) + ["-DB200_CSR_KERNEL=2", f"-DB200_WS_GATHER_WARPS={gw}",
                f"-DB200_WS_REDUCE_WARPS={rw}", f"-DB200_WS_REDUCE_GROUPS={rg}", f"-DB200_WS_STAGES={st}", f"-DB200_WS_GATHER_UNROLL={un}",
                f"-DB200_WS_MIN_CTAS={ct}"]
    if "RR" in v:
        return flags({k: x for k, x in v.items() if k not in ("RR", "RU")}) + [f"-DB200_CSR_RED_ROWS={v['RR']}", f"-DB200_CSR_RED_U={v['RU']}"]
    if "KERNEL" in v:
        extra = [f"-DB200_CSR_KERNEL={v['KERNEL']}"] + ([f"-DB200_CSR_PIPE_OFFS={v['OFFS']}"] if "OFFS" in v else [])
        return flags({k: x for k, x in v.items() if k not in ("KERNEL", "OFFS")}) + extra
    return [f"-DB200_CSR_TILE_ITEMS={v['TILE']}", f"-DB200_CSR_LONG_ROW={v['LONG']}", f"-DB200_CSR_BLOCK={v['BLOCK']}",
            f"-DB200_CSR_BATCH={v['BATCH']}", f"-DB200_CSR_MIN_CTAS={v['MIN']}"]


def build_flat_only(b, tag, extra, out):
    """The csr_flat_kernel tunables are read by spmv_csr_flat.cu alone: compile that file, link it with the default build's
    objects of every other file."""
    bdir = os.path.join(b.PKG_DIR, "build", "v_" + tag)
    os.makedirs(bdir, exist_ok=True)
    obj = os.path.join(bdir, "spmv_csr_flat.cu.o")
    cmd = [b.nvcc(), *b.NVCC_FLAGS, *extra, "-c", os.path.join(b.CSRC, "spmv_csr_flat.cu"), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    with open(os.path.join(bdir, "build.log"), "w") as f:
        f.write("$ " + " ".join(cmd) + "\n" + r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed on variant {tag}:\n{r.stdout}{r.stderr}")
    objs = [obj if s == "spmv_csr_flat.cu" else os.path.join(b.PKG_DIR, "build", s + ".o") for s in b.SOURCES]
    subprocess.run([b.nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", out, *objs, "-ldl", "-lpthread"], check=True)


def build():
    from concurrent.futures import ThreadPoolExecutor
    from cudalibrarysamples_b200 import build as b
    os.makedirs(VDIR, exist_ok=True)
    flat_only = {t: v for t, v in VARIANTS.items() if "FLATL1" in v}
    if flat_only:
        b.build_native()                                        # the objects the flat-only variants link against
        with ThreadPoolExecutor(os.cpu_count() or 4) as ex:
            list(ex.map(lambda tv: build_flat_only(b, tv[0], flags(tv[1]), os.path.join(VDIR, f"libb200spmv_{tv[0]}.so")),
                        flat_only.items()))
    for tag, v in VARIANTS.items():
        out = os.path.join(VDIR, f"libb200spmv_{tag}.so")
        if tag not in flat_only:
            b.build_native(extra_flags=flags(v), out_path=out, tag="v_" + tag)
        log = open(os.path.join(ROOT, "cudalibrarysamples_b200", "build", "v_" + tag, "build.log")).read()
        i = log.find("csr_short_kernelIdEE") if "SHORT" in v else log.find("csr_flat_kernelIdEE") if ("FLAT" in v or "FLAT3" in v or "FLATHOT" in v or "FLATL1" in v) else log.find("csr_seg_kernelIdEE") if "SEG" in v else log.find("csr_rowwise_kernelIdEE") if "RW" in v else log.find("csr_ws_kernelIdEE") if "WS" in v else max(log.find("csr_pipe_kernelIdEE"), log.find("csr_tile_kernelIdEE")) if "-DB200_CSR_KERNEL=0" not in " ".join(flags(v)) else log.find("csr_tile_kernelIdEE")
        regs = log[i:i + 400].split("Used ")[1].split(",")[0] if i >= 0 else "?"
        print(tag, regs)


def make_workload(name):
    import torch
    from cudalibrarysamples_b200 import workloads as W
    if name.endswith("_f32"):                                  # same structure, fp32 values
        rows, off, col, val = make_workload(name[:-4])
        return rows, off, col, val.float()
    if name.startswith("rmat"):
        rows = {"rmat1m": 1_000_000, "rmat10m": 10_000_000, "rmat4m": 4_000_000, "rmat250k": 250_000}[name]
        off, col, val = W.rmat_csr(rows)
    elif name == "uniform1m":
        rows = 1_000_000
        g = torch.Generator(device="cuda").manual_seed(1)
        col = torch.randint(0, rows, (rows, 16), device="cuda", generator=g, dtype=torch.int32).sort(dim=1).values.reshape(-1).contiguous()
        off = (torch.arange(rows + 1, device="cuda", dtype=torch.int64) * 16).to(torch.int32)
        val = W.uniform(43, rows * 16)
    elif name.startswith("stencil5_"):
        g = int(name.split("_")[1])
        rows = g * g
        off, col, val = W.stencil5_csr(g)
    elif name.startswith("laplace7_"):
        nx = int(name.split("_")[1])
        rows = nx ** 3
        off, col, val = W.laplace7_csr(nx)
    else:
        raise ValueError(name)
    return rows, off, col, val


def run(workloads, variants=None, steps=100):
    import torch
    from cudalibrarysamples_b200 import cusparse_api as cs
    from cudalibrarysamples_b200 import workloads as W
    results = {}
    libs = [("default", None)] + [(t, os.path.join(VDIR, f"libb200spmv_{t}.so")) for t in VARIANTS if (variants is None or t in variants)]
    libs = [(t, p) for t, p in libs if p is None or os.path.exists(p)]
    if os.environ.get("SWEEP_SET") == "kernels":     # every CSR kernel of the default library, picked through b200spmv_set_option
        libs = [("default", None)] + [("kernel:" + k, None) for k in ("flat", "short", "tile", "pipe", "seg", "seg:48", "rowwise")]
    for wl in workloads:
        rows, off, col, val = make_workload(wl)
        nnz = int(col.numel())
        x = W.uniform(44, rows, val.dtype)
        nbytes = W.csr_bytes(rows, rows, nnz, val.element_size())
        ref = None
        print(f"== {wl}: rows={rows} nnz={nnz} alg_bytes={nbytes / 1e6:.1f} MB", flush=True)
        order = libs + [("cusparse", "closed")]
        # SWEEP_ROUNDS > 1: the whole list again, every other round in reverse order, so that drift of the clock or of the
        # neighbours' load spreads over all variants; results then hold one entry per round
        rounds = int(os.environ.get("SWEEP_ROUNDS", "1"))
        for tag, path in [tp for r in range(rounds) for tp in (order if r % 2 == 0 else order[::-1])]:
            api = cs.Api("cusparse") if tag == "cusparse" else cs.Api("b200", lib_path=path)
            if tag != "cusparse":
                parts = tag.split(":") if tag.startswith("kernel:") else ["", "auto"]
                api.set_option("B200SPMV_FLAT", "on" if parts[1] == "flat" else "auto" if parts[1] == "auto" else "off")
                api.set_option("B200SPMV_SHORT", "on" if parts[1] == "short" else "auto" if parts[1] == "auto" else "off")
                api.set_option("B200SPMV_CSR_KERNEL", "auto" if parts[1] in ("flat", "short") else parts[1])
                api.set_option("B200SPMV_SEG_DENSE", parts[2] if len(parts) > 2 else "24")
            op = cs.SpMVOperator(api, "csr", rows, rows, dict(off=off, col=col, val=val))
            y = torch.zeros(rows, dtype=val.dtype, device="cuda")
            for _ in range(5):
                op(x, y, 1.0, 0.0)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                op(x, y, 1.0, 0.0)
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / steps
            if ref is None:
                ref = y.clone()
            err = float((torch.linalg.norm(y.double() - ref.double()) / torch.linalg.norm(ref.double())).item())
            same = bool(torch.equal(y, ref))
            print(f"  {tag:24s} {us:9.2f} us  {nbytes / us / 1e3:8.1f} GB/s  relerr_vs_first {err:.1e}  bits_equal {same}", flush=True)
            r = dict(us=us, gbs=nbytes / us / 1e3, err=err, bits_equal=same)
            if rounds > 1:
                results.setdefault(wl, {}).setdefault(tag, []).append(r)
            else:
                results.setdefault(wl, {})[tag] = r
            op.close()
        del off, col, val, x
        torch.cuda.empty_cache()
    return results


if __name__ == "__main__":
    if sys.argv[1] == "build":
        build()
    else:
        wls = sys.argv[2:] or ["rmat1m", "uniform1m", "stencil5_4096"]
        res = run(wls)
        os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
        json.dump(res, open(os.path.join(ROOT, "gpurun_out", "sweep.json"), "w"), indent=1)
