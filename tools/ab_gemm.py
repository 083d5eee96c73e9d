"""A/B timing of the GEMMs of the step between builds of libb200mdm.so of the same ABI.

    python tools/ab_gemm.py LIB_A LIB_B [LIB_C ...] [--rounds 3] [--json out.json]

Each library is loaded in its own child process (B200MDM_LIB) and the children run in turn, `--rounds` times, so that
clock and thermal drift fall on every build alike.  Every shape is timed through the kernel-test entry points
(b200mdm_test_gemm_f16 with block_n 128, b200mdm_test_gemm_epi, b200mdm_test_gemm_resid_ln), which launch the kernel the
step launches:
  warm     50 back-to-back launches captured in one CUDA graph (L2 warm: the operands stay resident), mean per launch,
           median of 5 replays
  flushed  one launch after writing a 256 MB buffer (evicts the 50 MB L2), median of 20
The report gives, per build and shape, the median over the rounds and the spread (min-max) of the per-round figures.
"""
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# name: (M, N, K, entry, mode) -- entry "f16": b200mdm_test_gemm_f16 with act = mode; "epi": b200mdm_test_gemm_epi
# with epi = mode (0: [hi | lo] + GELU, 1: per-column global bias); "ln": b200mdm_test_gemm_resid_ln (N = 512, in place
# on an [M, 1024] [hi | lo] residual stream; every launch re-normalises it, which leaves the timing unchanged)
SHAPES = {
    "c2 QKV":            (25216, 1536, 512, "f16", 0),
    "c2 FFN-up + GELU":  (25216, 1024, 512, "f16", 1),
    "DiP QKV":           (15360, 1536, 512, "f16", 0),
    "DiP Q (cross)":     (15360, 512, 512, "f16", 0),
    "DiP K/V all layers": (4096, 8192, 512, "epi", 1),
    "DiP FFN-up [hi|lo]": (15360, 1024, 1024, "epi", 0),
    "c2 out-proj + LN":  (25216, 512, 512, "ln", 0),
    "c2 FFN-down + LN":  (25216, 512, 1024, "ln", 0),
    "DiP cross out-proj + LN": (15360, 512, 512, "ln", 0),
    "DiP FFN-down + LN": (15360, 512, 2048, "ln", 0),
}


def child():
    import ctypes
    import torch
    sys.path.insert(0, ROOT)
    from b200mdm import _lib as L
    lib = L.load()
    torch.cuda.set_device(0)
    st = torch.cuda.Stream()
    out = {}
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, (M, N, K, entry, mode) in SHAPES.items():
        a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).half()
        w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).half()
        bias = torch.randn(N, device="cuda", generator=g)
        if entry == "ln":
            o = torch.randn(M, 2 * N, device="cuda", generator=g).half()
            gamma = 1 + 0.1 * torch.randn(N, device="cuda", generator=g)
            beta = 0.1 * torch.randn(N, device="cuda", generator=g)
            pg, pe = ctypes.c_void_p(gamma.data_ptr()), ctypes.c_void_p(beta.data_ptr())
        else:
            o = torch.empty(M, 2 * N if (entry == "epi" and mode == 0) else N, device="cuda", dtype=torch.float16)
        pa, pw, pb, po = (ctypes.c_void_p(t.data_ptr()) for t in (a, w, bias, o))

        def call():
            s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
            if entry == "f16":
                L.check(lib.b200mdm_test_gemm_f16(pa, pw, pb, po, M, N, K, mode, 128, s))
            elif entry == "ln":
                L.check(lib.b200mdm_test_gemm_resid_ln(pa, pw, pb, pg, pe, po, M, K, s))
            else:
                L.check(lib.b200mdm_test_gemm_epi(pa, pw, pb, po, M, N, K, mode, s))

        with torch.cuda.stream(st):
            for _ in range(3):
                call()
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=st):
                for _ in range(50):
                    call()
            warm = []
            for _ in range(6):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                graph.replay()
                e1.record(st)
                torch.cuda.synchronize()
                warm.append(e0.elapsed_time(e1) * 1e3 / 50)
            cold = []
            for _ in range(20):
                flush.add_(1)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                call()
                e1.record(st)
                torch.cuda.synchronize()
                cold.append(e0.elapsed_time(e1) * 1e3)
            del graph
        out[name] = {"warm_us": statistics.median(warm[1:]), "flushed_us": statistics.median(cold),
                     "tflops_warm": 2.0 * M * N * K / (statistics.median(warm[1:]) * 1e-6) / 1e12}
    print("AB_RESULT " + json.dumps(out))


def main():
    args = sys.argv[1:]
    rounds, jpath = 3, None
    if "--rounds" in args:
        i = args.index("--rounds")
        rounds = int(args[i + 1])
        del args[i:i + 2]
    if "--json" in args:
        i = args.index("--json")
        jpath = args[i + 1]
        del args[i:i + 2]
    libs = [os.path.abspath(p) for p in args]
    if len(libs) < 1:
        sys.exit(__doc__)
    res = {lib: [] for lib in libs}
    for r in range(rounds):
        for lib in libs:
            env = dict(os.environ, B200MDM_LIB=lib)
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=env, stdout=subprocess.PIPE,
                               stderr=subprocess.STDOUT, text=True)
            line = [ln for ln in p.stdout.splitlines() if ln.startswith("AB_RESULT ")]
            if p.returncode != 0 or not line:
                sys.stderr.write(p.stdout)
                sys.exit("child for %s failed (exit %d)" % (lib, p.returncode))
            res[lib].append(json.loads(line[0][len("AB_RESULT "):]))
            print("round %d done: %s" % (r + 1, lib), flush=True)
    summary = {}
    print("%-24s %-44s %28s %28s" % ("shape", "library", "warm us: median (min-max)", "flushed us: median (min-max)"))
    for name in SHAPES:
        for lib in libs:
            ws = [x[name]["warm_us"] for x in res[lib]]
            cs = [x[name]["flushed_us"] for x in res[lib]]
            summary.setdefault(name, {})[lib] = {"warm_us": ws, "flushed_us": cs}
            print("%-24s %-44s %8.1f (%6.1f-%6.1f)      %8.1f (%6.1f-%6.1f)" % (
                name, lib[-44:], statistics.median(ws), min(ws), max(ws), statistics.median(cs), min(cs), max(cs)))
    if jpath:
        with open(jpath, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    if sys.argv[1:] == ["--child"]:
        child()
    else:
        main()
