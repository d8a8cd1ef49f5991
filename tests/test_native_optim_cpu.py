"""The native optimizer step without a GPU: the argument checks and workspace size of b200kge_adagrad_step /
b200kge_sparse_adam_step through ctypes, the routing of `user.b200_native_optimizer` in the three training jobs, and
the host logic of kge_b200.optim (state, step counts, scalars, refusals, checkpoints) with the two engine entries
replaced by torch-formula stand-ins."""
import ctypes as C

import pytest
import torch

from kge_b200 import hostenv, optim


# ---- C ABI: argument checks (all before any launch) and the workspace size
@pytest.fixture(scope="module")
def lib():
    from kge_b200 import _lib

    try:
        return _lib.load()
    except OSError as e:
        pytest.skip(f"libb200kge.so not loadable here: {e}")


_BUF = (C.c_float * 64)()
_IDS = (C.c_int64 * 16)()


def _adagrad(lib, **over):
    a = dict(p=C.addressof(_BUF), s=C.addressof(_BUF), rows=4, dim=4, g=C.addressof(_BUF), gr=C.addressof(_IDS), nnz=3,
             coalesced=0, foreach=1, clr=0.1, eps=1e-10, wd=0.0, ws=C.addressof(_BUF), wsb=0)
    a.update(over)
    return lib.b200kge_adagrad_step(a["p"], a["s"], a["rows"], a["dim"], a["g"], a["gr"], a["nnz"], a["coalesced"],
                                    a["foreach"], a["clr"], a["eps"], a["wd"], a["ws"], a["wsb"], None)


def _sparse_adam(lib, **over):
    a = dict(p=C.addressof(_BUF), m=C.addressof(_BUF), q=C.addressof(_BUF), rows=4, dim=4, g=C.addressof(_BUF),
             gr=C.addressof(_IDS), nnz=3, coalesced=0, b1=0.1, b2=0.001, eps=1e-8, step=0.01, ws=C.addressof(_BUF),
             wsb=0)
    a.update(over)
    return lib.b200kge_sparse_adam_step(a["p"], a["m"], a["q"], a["rows"], a["dim"], a["g"], a["gr"], a["nnz"],
                                        a["coalesced"], a["b1"], a["b2"], a["eps"], a["step"], a["ws"], a["wsb"], None)


def _last_error(lib):
    return lib.b200kge_last_error().decode()


def test_adagrad_entry_refuses_bad_arguments(lib):
    from kge_b200._lib import ERR_INVALID as INVALID, ERR_UNSUPPORTED as UNSUPPORTED, ERR_WORKSPACE as WORKSPACE

    assert _adagrad(lib, p=None) == INVALID
    assert _adagrad(lib, s=None) == INVALID
    assert _adagrad(lib, g=None) == INVALID
    assert _adagrad(lib, gr=None, g=None) == INVALID            # dense gradient missing
    assert _adagrad(lib, rows=-1) == INVALID
    assert _adagrad(lib, dim=0) == INVALID
    assert _adagrad(lib, nnz=-1) == INVALID
    assert _adagrad(lib, wd=0.1, coalesced=1) == INVALID
    assert _last_error(lib) == "weight_decay option is not compatible with sparse gradients"
    assert _adagrad(lib, wsb=0) == WORKSPACE                     # uncoalesced: the row set needs a workspace
    assert _adagrad(lib, ws=None, wsb=1 << 20) == WORKSPACE
    assert _adagrad(lib, rows=1 << 31, wsb=1 << 40) == UNSUPPORTED


def test_sparse_adam_entry_refuses_bad_arguments(lib):
    from kge_b200._lib import ERR_INVALID as INVALID, ERR_WORKSPACE as WORKSPACE

    assert _sparse_adam(lib, gr=None) == INVALID
    assert _last_error(lib) == "SparseAdam does not support dense gradients, please consider Adam instead"
    assert _sparse_adam(lib, p=None) == INVALID
    assert _sparse_adam(lib, m=None) == INVALID
    assert _sparse_adam(lib, q=None) == INVALID
    assert _sparse_adam(lib, g=None) == INVALID
    assert _sparse_adam(lib, rows=-2) == INVALID
    assert _sparse_adam(lib, nnz=-1) == INVALID
    assert _sparse_adam(lib, wsb=0) == WORKSPACE


def test_optim_step_workspace_bytes(lib):
    def up(b):
        return (b + 255) // 256 * 256

    for rows, dim, nnz in ((4, 4, 3), (40943, 512, 1_026_048), (4_800_000, 512, 1_026_048), (10, 7, 1000)):
        cap = min(rows, nnz)
        row_set = up(rows * 4) + up(-(-rows // 4096) * 4)
        want = row_set + up(cap * 8) + 256 + up(cap * dim * 4)
        assert lib.b200kge_optim_step_workspace_bytes(rows, dim, nnz, 0) == want
        assert lib.b200kge_optim_step_workspace_bytes(rows, dim, nnz, 1) == 0
    assert lib.b200kge_optim_step_workspace_bytes(10, 4, 0, 0) == 0


# ---- host logic: the engine entries replaced by the torch formulas they implement
@pytest.fixture()
def stub(monkeypatch):
    """engine.adagrad_step / sparse_adam_step as torch's single-parameter formulas on CPU tensors; parameters on the
    CPU pass the device check.  Records every call's scalars."""
    from kge_b200 import engine

    calls = []

    @torch.no_grad()
    def adagrad_step(param, state_sum, grad, clr, eps, weight_decay=0.0, foreach_order=True):
        calls.append(dict(kind="adagrad", param=param, clr=clr, eps=eps, wd=weight_decay, foreach=foreach_order,
                          sparse=grad.is_sparse))
        if grad.is_sparse:
            g = grad.coalesce()
            i, v = g._indices()[0], g._values()
            state_sum[i] += v * v
            param[i] += -clr * (v / (state_sum[i].sqrt() + eps))
            return
        g = grad + weight_decay * param if weight_decay else grad
        state_sum.addcmul_(g, g)
        param.addcdiv_(g, state_sum.sqrt().add_(eps), value=-clr)

    @torch.no_grad()
    def sparse_adam_step(param, exp_avg, exp_avg_sq, grad, beta1, beta2, eps, step_size):
        calls.append(dict(kind="sparse_adam", param=param, step_size=step_size))
        g = grad.coalesce()
        i, v = g._indices()[0], g._values()
        if v.numel() == 0:
            return
        m0, q0 = exp_avg[i], exp_avg_sq[i]
        mu, qu = (v - m0) * (1 - beta1), (v * v - q0) * (1 - beta2)
        exp_avg[i] = m0 + mu
        exp_avg_sq[i] = q0 + qu
        param[i] += -step_size * ((mu + m0) / ((qu + q0).sqrt() + eps))

    monkeypatch.setattr(engine, "adagrad_step", adagrad_step)
    monkeypatch.setattr(engine, "sparse_adam_step", sparse_adam_step)
    monkeypatch.setattr(optim, "_on_cuda", lambda p: True)
    return calls


def _tables(seed=0, shapes=((30, 8), (5, 8))):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(s, generator=g).requires_grad_(True) for s in shapes]


def _grads(params, step, sparse, seed=0):
    """One gradient per parameter: dense, or an uncoalesced COO tensor of value rows with repeated ids."""
    g = torch.Generator().manual_seed(seed * 100 + step)
    out = []
    for p in params:
        if not sparse:
            out.append(torch.randn(p.shape, generator=g))
            continue
        idx = torch.randint(0, p.shape[0], (7,), generator=g)
        idx[3] = idx[0]
        out.append(torch.sparse_coo_tensor(idx[None], torch.randn((7, p.shape[1]), generator=g), p.shape))
    return out


def _run(opt, params, steps, sparse, first=0, seed=0):
    for k in range(first, first + steps):
        for p, g in zip(params, _grads(params, k, sparse, seed)):
            p.grad = g
        opt.step()


def _pair(cls, sparse, **kw):
    a, b = _tables(), _tables()
    torch_opt, native_opt = cls(a, **kw), cls(b, **kw)
    optim.install_native_step(native_opt)
    return (torch_opt, a), (native_opt, b)


def _same_state_dicts(x, y):
    sx, sy = x.state_dict(), y.state_dict()
    assert sx["param_groups"] == sy["param_groups"]
    assert sx["state"].keys() == sy["state"].keys()
    for k in sx["state"]:
        a, b = sx["state"][k], sy["state"][k]
        assert a.keys() == b.keys()
        for key in a:
            if torch.is_tensor(a[key]):
                assert torch.is_tensor(b[key]) and a[key].dtype == b[key].dtype and a[key].device == b[key].device
                assert a[key].shape == b[key].shape
                torch.testing.assert_close(a[key], b[key], rtol=1e-6, atol=1e-7)
            else:
                assert type(a[key]) is type(b[key]) and a[key] == b[key]


@pytest.mark.parametrize("cls,sparse,kw", [
    (torch.optim.Adagrad, False, dict(lr=0.1, lr_decay=0.05, weight_decay=0.01, initial_accumulator_value=0.2)),
    (torch.optim.Adagrad, False, dict(lr=0.1, foreach=False)),
    (torch.optim.Adagrad, True, dict(lr=0.1, lr_decay=0.05, eps=1e-6)),
    (torch.optim.SparseAdam, True, dict(lr=0.01, betas=(0.8, 0.99), eps=1e-6)),
])
def test_state_dict_matches_torch(stub, cls, sparse, kw):
    (t, a), (n, b) = _pair(cls, sparse, **kw)
    _run(t, a, 4, sparse)
    _run(n, b, 4, sparse)
    assert stub and optim.is_native(n) and not optim.is_native(t)
    _same_state_dicts(t, n)
    for x, y in zip(a, b):
        torch.testing.assert_close(x, y, rtol=1e-6, atol=1e-7)


def test_clr_includes_lr_decay_and_foreach_order(stub):
    p = _tables()
    opt = torch.optim.Adagrad([{"params": p[:1]}, {"params": p[1:], "foreach": False}], lr=0.3, lr_decay=0.25)
    optim.install_native_step(opt)
    _run(opt, p, 3, False)
    clrs = [c["clr"] for c in stub if c["param"] is p[0]]
    assert clrs == [0.3 / (1 + s * 0.25) for s in range(3)]
    assert [c["foreach"] for c in stub] == [True, False] * 3
    # a group with a sparse gradient takes the single-tensor order for its dense gradients too
    stub.clear()
    opt = torch.optim.Adagrad(p, lr=0.3)
    optim.install_native_step(opt)
    p[0].grad, p[1].grad = torch.ones(p[0].shape), _grads(p[1:], 0, True)[0]
    opt.step()
    assert [(c["foreach"], c["sparse"]) for c in stub] == [(False, False), (False, True)]


def test_lr_is_read_at_every_call(stub):
    p = _tables()
    opt = torch.optim.SparseAdam(p, lr=0.01, betas=(0.9, 0.999))
    optim.install_native_step(opt)
    sched = torch.optim.lr_scheduler.StepLR(opt, step_size=1, gamma=0.5)
    for k in range(3):
        _run(opt, p, 1, True, first=k)
        sched.step()
    sizes = [c["step_size"] for c in stub if c["param"] is p[0]]
    want = [0.01 * 0.5 ** t * (1 - 0.999 ** (t + 1)) ** 0.5 / (1 - 0.9 ** (t + 1)) for t in range(3)]
    assert sizes == pytest.approx(want, rel=1e-12)


@pytest.mark.parametrize("cls", [torch.optim.Adagrad, torch.optim.SparseAdam])
def test_grad_none_is_skipped(stub, cls):
    p = _tables()
    opt = cls(p, lr=0.1)
    optim.install_native_step(opt)
    for k in range(2):
        p[0].grad = _grads(p, k, True)[0]
        opt.step()
    assert all(c["param"] is p[0] for c in stub) and len(stub) == 2
    st = opt.state_dict()["state"]
    if cls is torch.optim.Adagrad:
        assert float(st[0]["step"]) == 2 and float(st[1]["step"]) == 0
    else:
        assert st[0]["step"] == 2 and 1 not in st


def _torch_error(opt, params, grads):
    for p, g in zip(params, grads):
        p.grad = g
    with pytest.raises(RuntimeError) as e:
        opt.step()
    return str(e.value)


def test_refusals_raise_torchs_errors(stub):
    (t, a), (n, b) = _pair(torch.optim.Adagrad, True, lr=0.1, weight_decay=0.1)
    want = _torch_error(t, a, _grads(a, 0, True))
    assert _torch_error(n, b, _grads(b, 0, True)) == want == "weight_decay option is not compatible with sparse gradients"
    (t, a), (n, b) = _pair(torch.optim.SparseAdam, False, lr=0.1)
    want = _torch_error(t, a, _grads(a, 0, False))
    assert _torch_error(n, b, _grads(b, 0, False)) == want and "does not support dense gradients" in want
    assert not stub


@pytest.mark.parametrize("cls,sparse,kw", [(torch.optim.Adagrad, False, dict(lr=0.1, lr_decay=0.1)),
                                           (torch.optim.Adagrad, True, dict(lr=0.1)),
                                           (torch.optim.SparseAdam, True, dict(lr=0.05))])
def test_checkpoint_round_trip(stub, cls, sparse, kw):
    """Two steps with the native step, resumed for two with torch's, and the reverse, against four of torch's."""
    ref = _tables()
    r = cls(ref, **kw)
    _run(r, ref, 4, sparse)
    for first_native in (True, False):
        p = _tables()
        opt = cls(p, **kw)
        if first_native:
            optim.install_native_step(opt)
        _run(opt, p, 2, sparse)
        saved = opt.state_dict()
        q = [x.detach().clone().requires_grad_(True) for x in p]
        resumed = cls(q, **kw)
        resumed.load_state_dict(saved)
        if not first_native:
            optim.install_native_step(resumed)
        _run(resumed, q, 2, sparse, first=2)
        _same_state_dicts(r, resumed)
        for x, y in zip(ref, q):
            torch.testing.assert_close(x, y, rtol=1e-6, atol=1e-7)


def test_install_refuses_what_it_cannot_serve(stub):
    p = _tables()
    for opt, why in ((torch.optim.Adam(p), "Adam"), (torch.optim.SGD(p, lr=0.1), "SGD"),
                     (torch.optim.Adagrad(p, maximize=True), "maximize"),
                     (torch.optim.Adagrad(p, differentiable=True), "differentiable"),
                     (torch.optim.Adagrad(p, fused=True), "fused"),
                     (torch.optim.SparseAdam(p, maximize=True), "maximize"),
                     (torch.optim.Adagrad([torch.zeros(3, 2, dtype=torch.float64, requires_grad=True)]), "float64"),
                     (torch.optim.Adagrad([torch.zeros(3, 2, dtype=torch.complex64, requires_grad=True)]), "complex"),
                     (torch.optim.Adagrad([torch.zeros(4, 3).t().requires_grad_(True)]), "non-contiguous")):
        with pytest.raises(NotImplementedError, match=why):
            optim.install_native_step(opt)
        assert "step" not in vars(opt)


def test_cpu_parameters_are_refused():
    with pytest.raises(NotImplementedError, match="cpu"):
        optim.install_native_step(torch.optim.Adagrad(_tables()))


# ---- routing in the three training jobs
E, R, D = 30, 4, 8
JOBS = {"1vsAll": "B200TrainingJob1vsAll", "KvsAll": "B200TrainingJobKvsAll",
        "negative_sampling": "B200TrainingJobNegativeSampling"}


@pytest.fixture()
def splits():
    if not hostenv.available():
        pytest.skip("reference not installed (oracle/install_ref.sh)")
    import jobs_util as ju

    return ju.synthetic_splits(E, R, 60, 10, 10)


def _job(splits, train_type, optimizer="Adagrad", option=True, extra=None):
    import jobs_util as ju

    ex = {"train.optimizer.default.type": optimizer, "user.b200_native_optimizer": option}
    if optimizer == "SparseAdam":
        ex["lookup_embedder.sparse"] = True
    ex.update(extra or {})
    return ju.make_job("b200_complex", E, R, D, splits, train_type=train_type, loss="kl", forward_only=False, extra=ex,
                       job_class=JOBS[train_type])


@pytest.mark.parametrize("train_type", list(JOBS))
def test_option_off_keeps_the_class_step(splits, train_type):
    job = _job(splits, train_type, option=False)
    assert "step" not in vars(job.optimizer) and not optim.is_native(job.optimizer)


@pytest.mark.parametrize("optimizer", ["Adagrad", "SparseAdam"])
@pytest.mark.parametrize("train_type", list(JOBS))
def test_option_on_patches_the_instance(splits, stub, train_type, optimizer):
    job = _job(splits, train_type, optimizer)
    assert type(job.optimizer) is getattr(torch.optim, optimizer)
    assert optim.is_native(job.optimizer) and "step" in vars(job.optimizer)
    assert job.optimizer.step.__self__ == job.optimizer


@pytest.mark.parametrize("train_type", list(JOBS))
def test_forward_only_jobs_are_untouched(splits, train_type):
    job = _job(splits, train_type, option=False)
    job.config.set("user.b200_native_optimizer", True)
    # parameters on the CPU: creating the job would raise if the option were applied
    fwd = type(job)(job.config, job.dataset, model=job.model, forward_only=True)
    assert fwd.is_forward_only and not hasattr(fwd, "optimizer")


@pytest.mark.parametrize("train_type", list(JOBS))
@pytest.mark.parametrize("optimizer,extra,why", [
    ("Adam", {}, "Adam"),
    ("Adagrad", {"train.optimizer.default.args.maximize": True}, "maximize"),
    ("Adagrad", {}, "cpu"),
])
def test_creation_refuses(splits, train_type, optimizer, extra, why, request):
    if why != "cpu":
        request.getfixturevalue("stub")
    with pytest.raises(NotImplementedError, match=f"user.b200_native_optimizer: .*{why}"):
        _job(splits, train_type, optimizer, extra=extra)
