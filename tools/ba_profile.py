"""Per-kernel device time of the local-BA try loop (CUDA events around every launch).  Run on the GPU box."""
import ctypes as C
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))
import ba_data  # noqa: E402
import conftest  # noqa: E402

plp = conftest.load_package()
from plpslam_b200.ba import LocalBA  # noqa: E402

ctx = plp.Context(0)
lib = plp.lib()
prob = ba_data.make_ba_problem(42)
st = prob.struct()
ba = LocalBA(ctx, st, (len(prob.kf_fixed), len(prob.pt_pos_w), len(prob.line_plucker), len(prob.pt_edge_kf),
                       len(prob.line_edge_kf)))
ba.bench_tries(15)
ctx._check(lib.plp_ctx_kernel_timing(ctx.handle, 1))
ba.bench_tries(30)
buf = C.create_string_buffer(1 << 16)
ctx._check(lib.plp_ctx_kernel_timing_report(ctx.handle, buf, C.c_size_t(len(buf))))
ctx._check(lib.plp_ctx_kernel_timing(ctx.handle, 0))
kt = json.loads(buf.value.decode())
tot = sum(v["total_ms"] for v in kt.values())
print(f"total {tot:.3f} ms for 31 tries -> {tot / 31 * 1e3:.1f} us/try")
for k, v in sorted(kt.items(), key=lambda kv: -kv[1]["total_ms"]):
    print(f"   {k:28s} n={v['count']:4d} mean_us={1e3 * v['total_ms'] / v['count']:8.1f} share={v['total_ms'] / tot:.3f}")
ba.close()
