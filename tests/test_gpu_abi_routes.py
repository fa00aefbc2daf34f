"""C-ABI routes of caller arrays: host (numpy) and device (torch CUDA) arrays, in every combination, give bitwise the same
outputs on fp64 and fp32 handles; host calls that span several chunks give the device call's outputs; and an fp32 handle
rejects bad arguments with the fp64 handle's exception and message."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F64, F32 = 0, 1
EI = 0
# (inputs on the device, outputs on the device)
ROUTES = [(False, False), (True, True), (True, False), (False, True)]


def _lib():
    from trieste_b200 import _lib

    return _lib


class In:
    """An input array, staged on the route's side."""

    def __init__(self, a):
        self.a = np.ascontiguousarray(a)


class Out:
    """An output array of the given shape and dtype, allocated on the route's side."""

    def __init__(self, shape, dtype):
        self.shape, self.dtype = shape, dtype


def _ptr(obj):
    return obj.data_ptr() if hasattr(obj, "data_ptr") else obj.ctypes.data


def _call(fn, args, route):
    """fn(*args) with In / Out arrays placed as `route` says; returns the outputs as numpy arrays."""
    import torch

    dev_in, dev_out = route
    keep, outs, cargs = [], [], []
    for a in args:
        if isinstance(a, In):
            obj = torch.from_numpy(a.a).cuda() if dev_in else a.a
        elif isinstance(a, Out):
            fill = -1 if np.dtype(a.dtype).kind == "i" else np.nan
            obj = np.full(a.shape, fill, dtype=a.dtype)
            if dev_out:
                obj = torch.from_numpy(obj).cuda()
            outs.append(obj)
        else:
            cargs.append(a)
            continue
        keep.append(obj)
        cargs.append(_ptr(obj))
    torch.cuda.synchronize()
    _lib().check(fn(*cargs))
    return [o.cpu().numpy() if hasattr(o, "cpu") else o for o in outs]


def _same_on_every_route(fn, args):
    ref = _call(fn, args, ROUTES[0])
    for route in ROUTES[1:]:
        got = _call(fn, args, route)
        for r, g in zip(ref, got):
            np.testing.assert_array_equal(g, r, err_msg=f"route {route}")
    return ref


def _data(N, D, seed, dt):
    rng = np.random.default_rng(seed)
    X = rng.uniform(size=(N, D)).astype(dt)
    y = (np.sin(3.0 * X).sum(1) + 0.1 * rng.standard_normal(N)).astype(dt)
    return X, y


class Handle:
    def __init__(self, dtype, N, D, seed=0, X=None, y=None):
        lib = _lib().lib()
        self.lib, self.dtype, self.D = lib, dtype, D
        self.dt = np.float32 if dtype == F32 else np.float64
        h = C.c_void_p()
        _lib().check(lib.tb_gp_create(C.byref(h), 0, dtype))
        self.h = h
        if X is None:
            X, y = _data(N, D, seed, self.dt)
        _lib().check(lib.tb_gp_set_data(h, _ptr(X), _ptr(y), N, D))
        ls = np.full(D, 0.4)
        _lib().check(lib.tb_gp_set_hyper(h, 3, 1.3, ls.ctypes.data_as(C.POINTER(C.c_double)), D, 1e-3, 0.1))
        _lib().check(lib.tb_gp_update_posterior_cache(h))

    def close(self):
        self.lib.tb_gp_destroy(self.h)


@pytest.fixture(params=[F64, F32], ids=["f64", "f32"])
def handle(request):
    hd = Handle(request.param, 300, 3)
    yield hd
    hd.close()


def test_every_dtype_dependent_call_is_the_same_on_every_route(handle):
    lib, h, D, dt = handle.lib, handle.h, handle.D, handle.dt
    rng = np.random.default_rng(1)
    M, B, q, S = 257, 19, 3, 64
    X = rng.uniform(size=(M, D)).astype(dt)
    Xb = rng.uniform(size=(B, q, D)).astype(dt)
    eps = rng.standard_normal((q, S)).astype(dt)
    w = rng.uniform(size=(q - 1, S))  # Sobol points: fp64 on every handle
    z = rng.standard_normal((S, M))  # standard-normal draws: fp64 on every handle
    eta = 0.5
    calls = {
        "get_cholesky": (lib.tb_gp_get_cholesky, [h, Out((300, 300), dt)]),
        "predict": (lib.tb_gp_predict, [h, In(X), M, Out(M, dt), Out(M, dt)]),
        "mean_gradient": (lib.tb_gp_mean_gradient, [h, In(X), M, Out(M, dt), Out((M, D), dt)]),
        "acq_eval": (lib.tb_acq_eval, [h, EI, eta, In(X), M, Out(M, dt), None]),
        "acq_eval_grad": (lib.tb_acq_eval, [h, EI, eta, In(X), M, Out(M, dt), Out((M, D), dt)]),
        "predict_joint": (lib.tb_gp_predict_joint, [h, In(Xb), B, q, Out((B, q), dt), Out((B, q, q), dt)]),
        "batch_mc_ei": (lib.tb_acq_batch_mc_ei, [h, In(Xb), B, q, In(eps), S, eta, 1e-6, Out(B, dt)]),
        "batch_mc_ei_grad": (lib.tb_acq_batch_mc_ei_grad, [h, In(Xb), B, q, In(eps), S, eta, 1e-6, Out(B, dt), Out((B, q, D), dt)]),
        "batch_ei": (lib.tb_acq_batch_ei, [h, In(Xb), B, q, In(w), S, eta, Out(B, dt)]),
        "batch_ei_grad": (lib.tb_acq_batch_ei_grad, [h, In(Xb), B, q, In(w), S, eta, Out(B, dt), Out((B, q, D), dt)]),
        "reparam_sample": (lib.tb_gp_reparam_sample, [h, In(Xb), B, q, In(eps), S, 1e-6, Out((B, S, q), dt)]),
        "covariance": (lib.tb_gp_covariance_between_points, [h, In(X[:40]), 40, In(X[40:100]), 60, Out((40, 60), dt)]),
        "sample_joint": (lib.tb_gp_sample_joint, [h, In(X), M, In(z), S, 1e-6, Out((S, M), dt)]),
    }
    for name, (fn, args) in calls.items():
        outs = _same_on_every_route(fn, args)
        for o in outs:
            assert o.dtype == dt and np.isfinite(o).all(), name
    # argmax: the winner is written to host scalars on every route
    ref = None
    for route in ROUTES:
        best = np.zeros(1, dt)
        idx = C.c_int64(-1)
        fn = lambda *a: lib.tb_acq_argmax(*a, best.ctypes.data, C.byref(idx))  # noqa: E731
        (vals,) = _call(fn, [h, EI, eta, In(X), M, Out(M, dt)], route)
        got = (vals.tobytes(), best.tobytes(), idx.value)
        ref = ref or got
        assert got == ref, route
    if dt == np.float64:
        assert ref[2] == int(np.argmax(np.frombuffer(ref[0], dt)))


@pytest.mark.parametrize("dtype", [F64, F32], ids=["f64", "f32"])
def test_set_and_append_data_are_the_same_on_every_route(dtype):
    import torch

    dt = np.float32 if dtype == F32 else np.float64
    X, y = _data(260, 4, 3, dt)
    chol = []
    for dev_in, _ in ROUTES[:2]:
        Xa, ya = (torch.from_numpy(X).cuda(), torch.from_numpy(y).cuda()) if dev_in else (X, y)
        torch.cuda.synchronize()
        hd = Handle(dtype, 256, 4, X=Xa[:256], y=ya[:256])
        try:
            _lib().check(hd.lib.tb_gp_append_data(hd.h, _ptr(Xa[256:]), _ptr(ya[256:]), 4))
            (L,) = _call(hd.lib.tb_gp_get_cholesky, [hd.h, Out((260, 260), dt)], (False, False))
            chol.append(L)
        finally:
            hd.close()
    np.testing.assert_array_equal(chol[0], chol[1])


def test_rff_topk_and_mvn_cdf_are_the_same_on_every_route():
    lib = _lib().lib()
    rng = np.random.default_rng(4)
    D, F, nb, M = 3, 96, 3, 1000
    r = C.c_void_p()
    _lib().check(lib.tb_rff_create(C.byref(r), 0))
    try:
        W = rng.standard_normal((F, D))
        b = rng.uniform(0, 2 * np.pi, F)
        ls = np.full(D, 0.3)
        theta = rng.standard_normal((nb, F))
        dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
        _lib().check(lib.tb_rff_set(r, dp(W), dp(b), F, D, dp(ls), 1.2, 0.1))
        _lib().check(lib.tb_rff_set_theta(r, dp(theta), nb))
        X = rng.uniform(size=(M, D))
        _same_on_every_route(lambda *a: lib.tb_rff_eval(*a, None, None), [r, In(X), M, Out((M, nb), np.float64)])
    finally:
        lib.tb_rff_destroy(r)
    v = rng.standard_normal(5000)
    k = 37
    fn = lambda dev, vals, M_, k_, tv, ti: lib.tb_topk(dev, F64, vals, M_, k_, tv, C.cast(C.c_void_p(ti), C.POINTER(C.c_int64)))  # noqa: E731
    tv, ti = _same_on_every_route(fn, [0, In(v), 5000, k, Out(k, np.float64), Out(k, np.int64)])
    np.testing.assert_array_equal(ti, np.argsort(-v, kind="stable")[:k])
    Bq, Q, S = 50, 4, 128
    x = rng.standard_normal((Bq, Q))
    mean = rng.standard_normal((Bq, Q))
    A = rng.standard_normal((Bq, Q, Q))
    cov = A @ A.transpose(0, 2, 1) + Q * np.eye(Q)
    w = rng.uniform(size=(Q - 1, S))
    _same_on_every_route(lib.tb_mvn_cdf, [0, In(x), In(mean), In(cov), Bq, Q, In(w), S, 0.0, Out(Bq, np.float64)])


def _launches(f):
    lib = _lib().lib()
    c0 = lib.tb_launch_count()
    f()
    return lib.tb_launch_count() - c0


def test_host_calls_spanning_several_chunks_match_device_calls():
    """Host arrays staged chunk by chunk through reused scratch, with one wait at the end of the call: the outputs equal
    the device call's, for each chunked driver, with at least two chunks and a partial last one."""
    hd = Handle(F64, 4096, 3)
    lib, h, D = hd.lib, hd.h, 3
    rng = np.random.default_rng(7)
    q, S = 3, 32
    eps = rng.standard_normal((q, S))
    try:
        M, M_eval = 150_001, 120_001  # mean_grad runs 65,536 points per launch; run_eval's chunks at N = 4096 are smaller
        X = rng.uniform(size=(M, D))
        B = 25_001  # q-batches; one chunk of the joint drivers at N = 4096 holds fewer
        Xb = rng.uniform(size=(B, q, D))
        w = rng.uniform(size=(q - 1, S))
        cases = {
            "eval values": (lib.tb_acq_eval, lambda m: [h, EI, 0.5, In(X[:m]), m, Out(m, np.float64), None], M_eval),
            "eval gradients": (lib.tb_acq_eval, lambda m: [h, EI, 0.5, In(X[:m]), m, Out(m, np.float64), Out((m, D), np.float64)],
                               M_eval),
            "mean gradient": (lib.tb_gp_mean_gradient, lambda m: [h, In(X[:m]), m, Out(m, np.float64), Out((m, D), np.float64)], M),
            "joint": (lib.tb_gp_predict_joint, lambda b: [h, In(Xb[:b]), b, q, Out((b, q), np.float64), Out((b, q, q), np.float64)], B),
            "qei grad": (lib.tb_acq_batch_mc_ei_grad,
                         lambda b: [h, In(Xb[:b]), b, q, In(eps), S, 0.5, 1e-6, Out(b, np.float64), Out((b, q, D), np.float64)], B),
            "batch mc ei": (lib.tb_acq_batch_mc_ei, lambda b: [h, In(Xb[:b]), b, q, In(eps), S, 0.5, 1e-6, Out(b, np.float64)], B),
            "reparam samples": (lib.tb_gp_reparam_sample,
                                lambda b: [h, In(Xb[:b]), b, q, In(eps), S, 1e-6, Out((b, S, q), np.float64)], B),
            "batch ei": (lib.tb_acq_batch_ei, lambda b: [h, In(Xb[:b]), b, q, In(w), S, 0.5, Out(b, np.float64)], B),
            "batch ei grad": (lib.tb_acq_batch_ei_grad,
                              lambda b: [h, In(Xb[:b]), b, q, In(w), S, 0.5, Out(b, np.float64), Out((b, q, D), np.float64)], B),
        }
        for name, (fn, args, n) in cases.items():
            _call(fn, args(1000), (True, True))  # lazy builds
            one = _launches(lambda: _call(fn, args(1000), (False, False)))
            host = []
            many = _launches(lambda: host.extend(_call(fn, args(n), (False, False))))
            assert many > one, name  # more than one chunk
            dev = _call(fn, args(n), (True, True))
            for a, b in zip(host, dev):
                np.testing.assert_array_equal(a, b, err_msg=name)
    finally:
        hd.close()
    # random-Fourier-feature trajectories: 2^22 candidates per chunk
    r = C.c_void_p()
    _lib().check(lib.tb_rff_create(C.byref(r), 0))
    try:
        F = 16
        dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
        W, b, ls, theta = rng.standard_normal((F, D)), rng.uniform(0, 6.28, F), np.full(D, 0.3), rng.standard_normal((1, F))
        _lib().check(lib.tb_rff_set(r, dp(W), dp(b), F, D, dp(ls), 1.0, 0.0))
        _lib().check(lib.tb_rff_set_theta(r, dp(theta), 1))
        m = (1 << 22) + 12_345
        Xr = rng.uniform(size=(m, D))
        fn = lambda *a: lib.tb_rff_eval(*a, None, None)  # noqa: E731
        one = _launches(lambda: _call(fn, [r, In(Xr[:1000]), 1000, Out((1000, 1), np.float64)], (False, False)))
        host = []
        many = _launches(lambda: host.extend(_call(fn, [r, In(Xr), m, Out((m, 1), np.float64)], (False, False))))
        assert many > one
        (dev,) = _call(fn, [r, In(Xr), m, Out((m, 1), np.float64)], (True, True))
        np.testing.assert_array_equal(host[0], dev)
    finally:
        lib.tb_rff_destroy(r)


def _error(fn):
    try:
        fn()
    except Exception as e:  # noqa: BLE001
        return type(e), str(e)
    return None


@pytest.mark.parametrize("case", ["negative count", "empty argmax", "zero dimension", "empty joint batch with bad q",
                                  "empty covariance set", "append nothing"])
def test_fp32_handles_reject_bad_arguments_as_fp64_handles_do(case):
    errors = []
    for dtype in (F64, F32):
        hd = Handle(dtype, 64, 2)
        lib, h, dt = hd.lib, hd.h, hd.dt
        X = np.zeros((8, 2), dt)
        out = np.zeros(64, dt)
        best, idx = np.zeros(1, dt), C.c_int64(0)
        calls = {
            "negative count": lambda: lib.tb_gp_predict(h, X.ctypes.data, -1, out.ctypes.data, out.ctypes.data),
            "empty argmax": lambda: lib.tb_acq_argmax(h, EI, 0.0, X.ctypes.data, 0, None, best.ctypes.data, C.byref(idx)),
            "zero dimension": lambda: lib.tb_gp_set_data(h, X.ctypes.data, out.ctypes.data, 8, 0),
            "empty joint batch with bad q": lambda: lib.tb_gp_predict_joint(h, None, 0, 0, None, None),
            "empty covariance set": lambda: lib.tb_gp_covariance_between_points(h, X.ctypes.data, 0, X.ctypes.data, 4,
                                                                                out.ctypes.data),
            "append nothing": lambda: lib.tb_gp_append_data(h, X.ctypes.data, out.ctypes.data, 0),
        }
        try:
            errors.append(_error(lambda: _lib().check(calls[case]())))
        finally:
            hd.close()
    assert errors[0] is not None and errors[0][0] is ValueError
    assert errors[1] == errors[0]
