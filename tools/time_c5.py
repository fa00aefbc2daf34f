"""Wall-clock timing of the C5 shape (N=8192, D=20, fp32 I/O): forward log-EI and value+gradient, several repetitions."""
import os, sys, time, math, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import __graft_entry__ as g
g.build()
import trieste_b200 as tb
from trieste_b200.acquisition import LogExpectedImprovement

def rff_obj(x, terms=64, seed=2):
    rng = np.random.default_rng(seed)
    w = rng.standard_normal((terms, x.shape[-1])) * 3.0
    ph = rng.uniform(0, 2 * math.pi, terms)
    a = rng.standard_normal(terms) / math.sqrt(terms)
    return (np.cos(x @ w.T + ph) * a).sum(-1, keepdims=True)

rng = np.random.default_rng(0)
X = rng.uniform(size=(8192, 20)).astype(np.float32)
y = rff_obj(X.astype(np.float64)).astype(np.float32)
ds = tb.Dataset(X, y)
m = tb.GaussianProcessRegression(tb.build_gpr(ds, tb.Box([0.0] * 20, [1.0] * 20)))
fn = LogExpectedImprovement().prepare_acquisition_function(m, ds)
xs = torch.rand(12_500, 1, 20, dtype=torch.float32, device="cuda")
xf = torch.rand(200_000, 1, 20, dtype=torch.float32, device="cuda")
out = {"engine_info": m.engine_info()}
for name, call in (("grad_ms", lambda: fn.value_and_gradient(xs)), ("forward_ms", lambda: fn(xf))):
    ts = []
    for _ in range(6):
        torch.cuda.synchronize(); t0 = time.perf_counter(); call(); torch.cuda.synchronize(); ts.append(1e3 * (time.perf_counter() - t0))
    out[name] = [round(t, 2) for t in ts]
print(json.dumps(out))
