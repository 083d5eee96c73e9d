"""Where the time of the fused residual + LayerNorm GEMM (gemm_resid_ln_cluster) goes, tile by tile.

    B200MDM_TRACE=1 python -m b200mdm.build     # -> motion-diffusion-model_b200/lib/libb200mdm_trace.so
    python tools/ln_phases.py [--lib PATH] [--runs 5] [--json out.json]

The instrumented library (-DB200_TRACE) stamps %globaltimer at fixed points of every tile: the producer thread and
one thread per consumer warpgroup write [CTA][tile iteration][role][event] into a device buffer, which
b200mdm_debug_ln_trace exposes.  Each shape runs through b200mdm_test_gemm_resid_ln, one launch after writing a 256 MB
buffer (the L2 is flushed, as it is for the residual stream between two of these launches in a step), `--runs` times.
The table gives the median over all (run, CTA, tile, warpgroup) of each phase, in microseconds:

  operand wait    tile start -> first k-block landed (A and W of the tile, loaded as ring stages free up)
  mainloop        first k-block landed -> last k-block's MMAs complete
  residual wait   last k-block complete -> first residual group landed
  residual rest   first -> last residual group landed (pass 1 runs in between)
  pass1+exchange  last residual group landed -> the peer CTA's row statistics have arrived
  pass2+stores    statistics -> the last group's LayerNorm written to shared memory (three groups stored meanwhile)
  last store      -> the last group's TMA store has read shared memory
  tile            tile start -> last store read
  producer: ring  producer tile start -> its first k-block load issued (waits for the previous tile's stores)
The globaltimer ticks in steps of up to 1 us on some parts, so single phases below that are coarse; medians over
thousands of tiles still order them.
"""
import ctypes
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# name: (M, K) -- the c2 step (128 packed CFG sequences x 197 tokens) and the DiP decoder (256 x 60)
SHAPES = {
    "c2 out-proj":       (25216, 512),
    "c2 FFN-down":       (25216, 1024),
    "DiP cross out-proj": (15360, 512),
    "DiP self out-proj":  (15360, 1024),
    "DiP FFN-down":      (15360, 2048),
}
# consumer events (roles 1, 2) and producer events (role 0), in the order the kernel stamps them
C_START, C_KB0, C_KBLAST, C_RES0, C_RESLAST, C_XCHG, C_PASS2, C_STORE = range(8)
P_START, P_KB0, P_RES = range(3)
PHASES = [("operand wait", C_START, C_KB0), ("mainloop", C_KB0, C_KBLAST), ("residual wait", C_KBLAST, C_RES0),
          ("residual rest", C_RES0, C_RESLAST), ("pass1+exchange", C_RESLAST, C_XCHG), ("pass2+stores", C_XCHG, C_PASS2),
          ("last store", C_PASS2, C_STORE), ("tile", C_START, C_STORE)]


def main():
    args = sys.argv[1:]
    runs, jpath = 5, None
    lib_path = os.path.join(ROOT, "motion-diffusion-model_b200", "lib", "libb200mdm_trace.so")
    for flag in ("--runs", "--json", "--lib"):
        if flag in args:
            i = args.index(flag)
            v = args[i + 1]
            del args[i:i + 2]
            if flag == "--runs":
                runs = int(v)
            elif flag == "--json":
                jpath = v
            else:
                lib_path = os.path.abspath(v)
    if not os.path.exists(lib_path):
        sys.exit("%s is missing: build it with B200MDM_TRACE=1 python -m b200mdm.build" % lib_path)
    os.environ["B200MDM_LIB"] = lib_path
    import numpy as np
    import torch
    sys.path.insert(0, ROOT)
    from b200mdm import _lib as L
    lib = L.load()
    if not hasattr(lib, "b200mdm_debug_ln_trace"):
        sys.exit("%s is not an instrumented build (no b200mdm_debug_ln_trace)" % lib_path)
    lib.b200mdm_debug_ln_trace.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int32)]
    torch.cuda.set_device(0)
    dims = (ctypes.c_int32 * 4)()
    L.check(lib.b200mdm_debug_ln_trace(None, dims))
    ctas, iters, roles, events = list(dims)
    host = np.zeros(ctas * iters * roles * events, dtype=np.uint64)

    def read_and_clear():
        L.check(lib.b200mdm_debug_ln_trace(host.ctypes.data_as(ctypes.c_void_p), dims))
        ns = host.astype(np.int64)
        hit = ns > 0   # slots the launch did not reach stay 0
        base = ns[hit].min() - 1 if hit.any() else 0   # relative to the launch, so that float64 keeps every nanosecond
        return np.where(hit, ns - base, 0).astype(np.float64).reshape(ctas, iters, roles, events)

    props = torch.cuda.get_device_properties(0)
    print("device: %s, %d SMs" % (props.name, props.multi_processor_count))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    report = {}
    for name, (M, K) in SHAPES.items():
        a = (torch.randn(M, K, device="cuda", generator=g) * 0.5).half()
        w = (torch.randn(512, K, device="cuda", generator=g) / K ** 0.5).half()
        vec = [torch.randn(512, device="cuda", generator=g) * 0.1 for _ in range(3)]
        hres = torch.randn(M, 1024, device="cuda", generator=g).half()
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

        def call():
            L.check(lib.b200mdm_test_gemm_resid_ln(p(a), p(w), p(vec[0]), p(vec[1]), p(vec[2]), p(hres), M, K, stream))

        for _ in range(3):
            call()
        torch.cuda.synchronize()
        samples = {ph: [] for ph, _, _ in PHASES}
        samples["producer: ring"] = []
        spans = []
        for _ in range(runs):
            flush.add_(1)
            torch.cuda.synchronize()
            read_and_clear()
            call()
            torch.cuda.synchronize()
            t = read_and_clear()
            cons = t[:, :, 1:, :].reshape(-1, events)
            cons = cons[(cons > 0).all(axis=1)]
            for ph, e0, e1 in PHASES:
                samples[ph].extend(((cons[:, e1] - cons[:, e0]) * 1e-3).tolist())
            prod = t[:, :, 0, :].reshape(-1, events)
            prod = prod[(prod[:, :P_RES + 1] > 0).all(axis=1)]
            samples["producer: ring"].extend(((prod[:, P_KB0] - prod[:, P_START]) * 1e-3).tolist())
            spans.append((cons[:, C_STORE].max() - min(cons[:, C_START].min(), prod[:, P_START].min())) * 1e-3)
        report[name] = {ph: statistics.median(v) for ph, v in samples.items()}
        report[name]["stamped span"] = statistics.median(spans)
        report[name]["tiles per CTA"] = int(t[:, :, 1, C_START].astype(bool).sum(axis=1).max())
    names = list(report)
    rows = [ph for ph, _, _ in PHASES] + ["producer: ring", "stamped span"]
    print("median per tile, us (flushed L2, %d runs)" % runs)
    print("%-16s" % "phase" + "".join("%20s" % nm for nm in names))
    for r in rows:
        print("%-16s" % r + "".join("%20.2f" % report[nm][r] for nm in names))
    print("%-16s" % "tiles per CTA" + "".join("%20d" % report[nm]["tiles per CTA"] for nm in names))
    if jpath:
        with open(jpath, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
