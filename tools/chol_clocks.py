"""SM-clock breakdown of ba_cholesky_kernel at window sizes, cycles per call as thread 0 sees them: load / factorisation (warp 0's
diagonal blocks) / panel + head block (all warps) / wait (warp 0 waiting for the trailing update) / backward / total.
The load phase (the resident kernel's copy of the envelope into shared memory by warps 1..7) overlaps warp 0's first diagonal block."""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lvio_fusion_b200 import _capi, backend, synth
lvb = _capi.load(); ctx = backend.Context(lvb)
for nk, nl in ((10, 4000), (20, 8000)):
    d = synth.make_ba_problem(nk, nl, with_imu=True)
    p = backend.Problem.from_dict(ctx, d)
    p.solve(max_num_iterations=3)
    out = (ctypes.c_longlong * 8)()
    lvb.check(lvb.debug_cholesky_clocks(out, 1), "clocks")
    p.update_params(d["poses"], d["vec3"], d["rho"])
    p.solve(max_num_iterations=10, function_tolerance=0.0, gradient_tolerance=0.0, parameter_tolerance=0.0)
    lvb.check(lvb.debug_cholesky_clocks(out, 1), "clocks")
    c = max(1, out[5])
    print("n=%d calls=%d (resident %d)  load %.0f  factorisation %.0f  panel+head %.0f  wait %.0f  backward %.0f  total %.0f cycles/call"
          % (p.dims()[0], c, out[7], out[6] / max(1, out[7]), out[0] / c, out[1] / c, out[2] / c, out[3] / c, out[4] / c))
