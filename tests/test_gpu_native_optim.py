"""The native optimizer step on the H100 (b200kge_adagrad_step, b200kge_sparse_adam_step) against torch's own
optimizers: one step from identical (p, state, grad) for dense Adagrad in both of torch's orders and for row-sparse
Adagrad and SparseAdam with coalesced, uncoalesced, full and empty gradients; a 20-step trajectory with a scheduler;
and the three training jobs with `user.b200_native_optimizer` against the same seeded jobs without it, checkpoints
included."""
import pytest
import torch

from kge_b200 import hostenv, optim

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from kge_b200 import engine

    if not torch.cuda.is_available() or not engine.device_ok():
        pytest.skip("needs an sm_90 device")
    return engine


def _bar(name, native, ref, before):
    """|native - torch| <= 4 * 2^-24 * (|x_torch| + |dx_torch|) per element; prints the non-bitwise count."""
    ref64, d = ref.double(), (ref.double() - before.double()).abs()
    err = (native.double() - ref64).abs()
    bound = 4 * 2.0 ** -24 * (ref64.abs() + d)
    diff = int((native != ref).sum())
    print(f"{name}: {diff} of {ref.numel()} elements not bitwise equal, max |d| {float(err.max()):.3e}")
    bad = err > bound
    assert not bad.any(), f"{name}: {int(bad.sum())} elements beyond the bar, worst {float((err - bound).max()):.3e}"
    return diff


def _state_tensors(opt, p):
    st = opt.state[p]
    return [st[k] for k in ("sum", "exp_avg", "exp_avg_sq") if k in st]


def _one_step(cls, shape, grad_fn, kw, state_init=None, seed=0):
    """One step of torch's optimizer and of the native one from identical (p, state, grad); returns, per tensor,
    (name, native, torch, before)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    p0 = torch.randn(shape, device="cuda", generator=g)
    grad = grad_fn(p0, g)
    out = []
    opts = []
    for native in (False, True):
        p = p0.clone().requires_grad_(True)
        opt = cls([p], **kw)
        if native:
            optim.install_native_step(opt)
        if state_init is not None:
            state_init(opt, p, torch.Generator(device="cuda").manual_seed(seed + 1))
        before = [t.clone() for t in _state_tensors(opt, p)]
        p.grad = grad.clone()
        opt.step()
        opts.append((p.detach(), _state_tensors(opt, p), before))
    (pt, st, sb), (pn, sn, _) = opts
    out.append(("param", pn, pt, p0))
    for k, (a, b, c) in enumerate(zip(sn, st, sb)):
        out.append((f"state{k}", a, b, c))
    return out


def _adagrad_state(steps):
    def init(opt, p, g):
        st = opt.state[p]
        st["sum"].add_(torch.rand(p.shape, device="cuda", generator=g))
        st["step"].fill_(steps)
    return init


def _adam_state(steps):
    def init(opt, p, g):
        st = opt.state[p]
        st["step"] = steps
        st["exp_avg"] = 0.1 * torch.randn(p.shape, device="cuda", generator=g)
        st["exp_avg_sq"] = 0.01 * torch.rand(p.shape, device="cuda", generator=g)
    return init


def _dense(p, g):
    return torch.randn(p.shape, device="cuda", generator=g)


DENSE_KW = [dict(lr=0.1), dict(lr=0.05, lr_decay=0.01, weight_decay=1e-3, eps=1e-6, initial_accumulator_value=0.1)]


@pytest.mark.parametrize("foreach", [None, False])
@pytest.mark.parametrize("kw", DENSE_KW)
@pytest.mark.parametrize("shape", [(14541, 512), (1_000_000, 512), (1000, 1), (1001, 7), (999, 130)])
def test_dense_adagrad_one_step(eng, shape, kw, foreach):
    for name, native, ref, before in _one_step(torch.optim.Adagrad, shape, _dense, dict(kw, foreach=foreach),
                                               _adagrad_state(3)):
        _bar(f"adagrad {shape} {kw} foreach={foreach} {name}", native, ref, before)


def _coalesced(rows):
    def fn(p, g):
        idx = torch.randperm(p.shape[0], device="cuda", generator=g)[:rows].sort().values
        return torch.sparse_coo_tensor(idx[None], torch.randn((rows, p.shape[1]), device="cuda", generator=g),
                                       p.shape).coalesce()
    return fn


def _uncoalesced(p, g):
    """S slot + O slot + penalty: three coalesced parts over overlapping rows, concatenated (autograd's sum).  The values
    lie on a 2^-12 grid, so the duplicates' sum is exact in every order and torch's coalesce() and the native one agree."""
    parts = [_coalesced(n)(p, g) for n in (3000, 2500, 800)]
    idx = torch.cat([x.indices() for x in parts], 1)
    vals = torch.cat([x.values() for x in parts]).mul(4096).round().div(4096)
    out = torch.sparse_coo_tensor(idx, vals, p.shape)
    assert not out.is_coalesced()
    return out


def _every_row(p, g):
    return _coalesced(p.shape[0])(p, g)


def _empty(p, g):
    return torch.sparse_coo_tensor(torch.zeros((1, 0), dtype=torch.int64, device="cuda"),
                                   torch.zeros((0, p.shape[1]), device="cuda"), p.shape)


SPARSE = {"coalesced": _coalesced(2000), "uncoalesced": _uncoalesced, "every_row": _every_row, "empty": _empty}
OPTS = {"adagrad": (torch.optim.Adagrad, dict(lr=0.1, lr_decay=0.01, eps=1e-8), _adagrad_state(2)),
        "sparse_adam": (torch.optim.SparseAdam, dict(lr=0.01, betas=(0.85, 0.995), eps=1e-6), _adam_state(4))}


@pytest.mark.parametrize("shape", [(40943, 128), (5000, 7)])
@pytest.mark.parametrize("grad", list(SPARSE))
@pytest.mark.parametrize("opt", list(OPTS))
def test_sparse_one_step(eng, opt, grad, shape):
    cls, kw, init = OPTS[opt]
    for name, native, ref, before in _one_step(cls, shape, SPARSE[grad], kw, init):
        _bar(f"{opt} {grad} {shape} {name}", native, ref, before)
        assert torch.equal(native, ref), f"{name}: not bitwise torch's"


@pytest.mark.parametrize("opt,grad", [("adagrad_dense", None), ("adagrad", "uncoalesced"),
                                      ("sparse_adam", "uncoalesced"), ("sparse_adam", "coalesced")])
def test_trajectory_with_scheduler(eng, opt, grad):
    """20 steps, lr halved after 10 by a StepLR: the final tables within 1e-6 of the table rms of torch's."""
    shape = (20000, 64)
    if opt == "adagrad_dense":
        cls, kw, fn = torch.optim.Adagrad, dict(lr=0.1, lr_decay=0.01, weight_decay=1e-4), _dense
    else:
        cls, kw, _ = OPTS[opt]
        fn = SPARSE[grad]
    g0 = torch.Generator(device="cuda").manual_seed(5)
    p0 = torch.randn(shape, device="cuda", generator=g0)
    finals = []
    for native in (False, True):
        p = p0.clone().requires_grad_(True)
        o = cls([p], **kw)
        if native:
            optim.install_native_step(o)
        sched = torch.optim.lr_scheduler.StepLR(o, step_size=10, gamma=0.5)
        g = torch.Generator(device="cuda").manual_seed(6)
        for _ in range(20):
            p.grad = fn(p0, g)
            o.step()
            sched.step()
        finals.append([p.detach()] + _state_tensors(o, p))
    for k, (a, b) in enumerate(zip(*finals)):
        rms = float(b.double().pow(2).mean().sqrt())
        err = float((a.double() - b.double()).abs().max())
        assert err <= 1e-6 * rms, f"tensor {k}: max|d| {err:.3e}, rms {rms:.3e}"


# ---- the jobs: two epochs with the option on against the same seeded job with it off
needs_ref = pytest.mark.skipif(not hostenv.available(), reason="reference not installed (oracle/install_ref.sh)")
E, R, D = 120, 6, 32
JOBS = {"1vsAll": "B200TrainingJob1vsAll", "KvsAll": "B200TrainingJobKvsAll",
        "negative_sampling": "B200TrainingJobNegativeSampling"}


@pytest.fixture(scope="module")
def splits():
    import jobs_util as ju

    return ju.synthetic_splits(E, R, 400, 20, 20)


def _make(splits, model, train_type, extra, option):
    import jobs_util as ju

    ex = dict(extra, **{"user.b200_native_optimizer": option})
    return ju.make_job("b200_" + model, E, R, D, splits, device="cuda", train_type=train_type, loss="kl",
                       batch_size=64, forward_only=False, extra=ex, job_class=JOBS[train_type])


def _epoch(job, ep):
    import jobs_util as ju

    job.epoch += 1
    if job.loader is None:
        job._prepare()
    ju.seed_all(10 + ep)
    return job.run_epoch()["avg_loss"]


def _compare_tables(a, b, what):
    for k, (x, y) in enumerate(zip(a.model.parameters(), b.model.parameters())):
        rms = float(y.detach().double().pow(2).mean().sqrt())
        err = float((x.detach().double() - y.detach().double()).abs().max())
        assert err <= 1e-5 * rms, f"{what}: parameter {k} max|d| {err:.3e}, rms {rms:.3e}"


def _replay(src, dst):
    """dst's optimizer steps with the gradients src's had at the same step.  The backward's atomics would otherwise make
    the two runs' gradients differ in the last bits, which Adagrad's first steps magnify; so the comparison is of the
    optimizer steps and the job's plumbing around them."""
    seen, s_step, d_step = [], src.optimizer.step, dst.optimizer.step

    def record(*a, **kw):
        seen.append([None if p.grad is None else p.grad.clone() for p in src.model.parameters()])
        return s_step(*a, **kw)

    def replay(*a, **kw):
        for p, g in zip(dst.model.parameters(), seen.pop(0)):
            p.grad = g
        return d_step(*a, **kw)
    src.optimizer.step, dst.optimizer.step = record, replay


def _job_pair(splits, model, train_type, extra, epochs=2):
    jobs = {}
    for option in (False, True):
        torch.manual_seed(0)
        jobs[option] = _make(splits, model, train_type, extra, option)
        assert optim.is_native(jobs[option].optimizer) == option
    with torch.no_grad():
        for a, b in zip(jobs[False].model.parameters(), jobs[True].model.parameters()):
            b.copy_(a)
    _replay(jobs[False], jobs[True])
    losses = {opt: [_epoch(job, ep) for ep in range(epochs)] for opt, job in jobs.items()}
    assert losses[True] == pytest.approx(losses[False], rel=1e-5), losses
    _compare_tables(jobs[True], jobs[False], f"{model} {train_type} {extra}")
    return jobs


ADAGRAD = {"train.optimizer.default.type": "Adagrad", "train.optimizer.default.args.lr": 0.2,
           "train.optimizer.default.args.weight_decay": 1e-4, "train.optimizer.default.args.lr_decay": 0.01}


@needs_ref
@pytest.mark.parametrize("train_type", ["1vsAll", "KvsAll"])
def test_1vsall_kvsall_jobs(eng, splits, train_type):
    _job_pair(splits, "complex", train_type, ADAGRAD)


NS = {"negative_sampling.num_samples.s": 5, "negative_sampling.num_samples.o": 7, "train.loss_arg": 1.0}
NS_OPT = {"adagrad_dense": {"train.optimizer.default.type": "Adagrad", "train.optimizer.default.args.lr": 0.2},
          "adagrad_sparse": {"train.optimizer.default.type": "Adagrad", "train.optimizer.default.args.lr": 0.2,
                             "lookup_embedder.sparse": True},
          "sparse_adam": {"train.optimizer.default.type": "SparseAdam", "train.optimizer.default.args.lr": 0.01,
                          "lookup_embedder.sparse": True}}
NS_EXTRA = {"plain": {},
            "weighted_lp": {"lookup_embedder.regularize": "lp", "lookup_embedder.regularize_weight": 1e-2,
                            "lookup_embedder.regularize_args.weighted": True},
            "unweighted_lp": {"lookup_embedder.regularize": "lp", "lookup_embedder.regularize_weight": 1e-2,
                              "lookup_embedder.regularize_args.weighted": False},
            "subbatch": {"train.subbatch_size": 24}}


@needs_ref
@pytest.mark.parametrize("extra", list(NS_EXTRA))
@pytest.mark.parametrize("opt", list(NS_OPT))
@pytest.mark.parametrize("model", ["complex", "rotate"])
def test_negative_sampling_jobs(eng, splits, model, opt, extra):
    _job_pair(splits, model, "negative_sampling", dict(NS, **NS_OPT[opt], **NS_EXTRA[extra]))


@needs_ref
@pytest.mark.parametrize("train_type,extra", [("1vsAll", ADAGRAD), ("negative_sampling", dict(NS, **NS_OPT["sparse_adam"])),
                                              ("negative_sampling", dict(NS, **NS_OPT["adagrad_sparse"]))])
def test_checkpoint_resumes_across_the_option(eng, splits, tmp_path, train_type, extra):
    """One epoch with the option on, checkpoint, resumed with it off (and the reverse): the second epoch matches the
    job that kept its option."""
    for first in (True, False):
        torch.manual_seed(0)
        job = _make(splits, "complex", train_type, extra, first)
        _epoch(job, 0)
        path = str(tmp_path / f"ckpt_{first}.pt")
        job.save(path)
        ckpt = torch.load(path, map_location="cuda", weights_only=False)     # holds the job's Config
        ckpt["file"] = path
        resumed = _make(splits, "complex", train_type, extra, not first)
        resumed.model.load_state_dict(job.model.state_dict())
        resumed._load(ckpt)
        assert optim.is_native(resumed.optimizer) == (not first)
        _replay(job, resumed)
        a, b = _epoch(job, 1), _epoch(resumed, 1)
        assert a == pytest.approx(b, rel=1e-5)
        _compare_tables(resumed, job, f"resumed with the option {'off' if first else 'on'}")
