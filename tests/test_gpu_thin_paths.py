"""The thin-channel kernels (thin.cu) and the glue kernels of a training step, called through the C ABI at their edge
shapes and compared with a float64 NumPy / SciPy product:

- thin_fwd_kernel: every term F <= 4, 16 <= ncols <= 128 (encoder / discriminator conv1, data gradients of the
  thin-output layers); vec4 and scalar column paths, condition slots over tiles that span many samples, the LINEAR /
  SLOPE / DUALMASK epilogues, and the eligibility limits of the condition staging buffer;
- thin_dw_kernel<4|8|12|16> + reduce_splits_kernel: weight gradients with F <= 4, the single- and multi-term forms, the
  operand swap of the thin-output layers (dw_col_stride), workspace-limited block counts;
- thinout_project_kernel + thinout_combine_kernel: <= 4 output columns, the project kernel's lane split and
  grid-stride loop, condition slots, bias, activation;
- cape_colsum, cape_resample with a condition, cape_gemm_batch.

Every case checks which kernels ran (CUDA activity tracing and cape_launch_count), that every element it should write
is finite and within 1e-4 of max |truth|, and that sentinels around and after its outputs are untouched.  Calls the
thin kernels reject are checked to take the generic kernels and still give the float64 result."""
import contextlib

import numpy as np
import pytest
import scipy.sparse as sp
import torch

pytestmark = pytest.mark.gpu

TOL = 1e-4
GUARD = 67            # sentinel floats after every output buffer
NAN = np.float32("nan")
ACTS = {"none": (0, 0.2), "leaky": (1, 0.2), "leaky.37": (1, 0.37), "relu": (2, 0.2)}
THIN = ("thin_fwd_kernel", "thin_dw_kernel", "thinout_project_kernel", "thinout_combine_kernel")


def _E():
    from cape_b200 import engine
    return engine


def _lib():
    from cape_b200 import _lib
    return _lib.load()


def _dev():
    return torch.device("cuda", 0)


def _tp():
    from cape_b200 import ops
    return ops.topology_for(_dev())


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@contextlib.contextmanager
def _knobs(tuning=(), tc=None):
    """Sets process-wide kernel-selection knobs for the duration of a block and always restores them."""
    lib, undo = _lib(), []
    try:
        for k, v in tuning:
            prev = lib.cape_set_tuning(k, v)
            undo.append(lambda k=k, prev=prev: lib.cape_set_tuning(k, prev))
        if tc is not None:
            prev = lib.cape_set_tensor_cores(1 if tc else 0)
            undo.append(lambda prev=prev: lib.cape_set_tensor_cores(prev))
        yield
    finally:
        for u in reversed(undo):
            u()


def _short(name):
    """'void cape::(anonymous namespace)::thin_dw_kernel<12>(cape::...)' -> 'thin_dw_kernel<12>'."""
    s = name.replace("(anonymous namespace)::", "")
    return s.split("(")[0].split("::")[-1].strip()


def _traced(fn, reset, attempts=3):
    """Runs fn() under CUDA activity tracing; returns the short names of the library's kernels it launched, in order,
    checked against the library's own launch counter.  A trace now and then lacks the record of the first kernel
    launched after tracing starts, so a torch kernel goes first; if records are still missing, reset() restores the
    outputs and the call runs again, and after `attempts` incomplete traces the case fails (the kernel selection could
    not be checked)."""
    from torch.profiler import ProfilerActivity, profile
    lib = _lib()
    for _ in range(attempts):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.zeros(1, device=_dev())
            torch.cuda.synchronize()
            n0 = lib.cape_launch_count()
            fn()
            torch.cuda.synchronize()
            launched = lib.cape_launch_count() - n0
        events = [e.name() for e in prof.profiler.kineto_results.events()]
        names = [_short(n) for n in events if "cape::" in n]
        if names and len(names) == launched:
            return names
        print("incomplete trace (%d launches counted, kernels %s): again" % (launched, names))
        reset()
        torch.cuda.synchronize()
    pytest.fail("the CUDA profiler recorded %d of the %d kernels launched in each of %d traces: cannot tell which "
                "kernels ran" % (len(names), launched, attempts))


def _ran(names, kernel):
    return any(n == kernel or n.startswith(kernel + "<") for n in names)


def _expect(names, kernels=(), launches=None, thin=None):
    """kernels: names (or template names) that must be among the launches; thin=False: none of the thin kernels ran."""
    for k in kernels:
        assert _ran(names, k), "expected %s, launched %s" % (k, names)
    if launches is not None:
        assert len(names) == launches, (names, launches)
    if thin is False:
        assert not any(_ran(names, k) for k in THIN), "a thin kernel ran: %s" % names


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def _check(got, init, mask, want, what=""):
    """got / init / want: flat float arrays of a whole buffer; mask: the elements the call writes.  Returns the
    relative error over the written elements."""
    assert np.isfinite(got[mask]).all(), "%s: %d elements left unwritten or non-finite" % (
        what, int((~np.isfinite(got[mask])).sum()))
    err = _rel(got[mask].astype(np.float64), want[mask])
    assert err < TOL, "%s: relative error %.3e" % (what, err)
    assert np.array_equal(got[~mask], init[~mask], equal_nan=True), "%s: wrote outside its target (%d elements)" % (
        what, int((~((got[~mask] == init[~mask]) | (np.isnan(got[~mask]) & np.isnan(init[~mask])))).sum()))
    return err


def _report(case, err):
    print("worst-rel-err %-60s %.3e" % (case, err))


def _operator(rng, rows_out, rows_in, width=7, empty_every=13):
    """A random sparse [rows_out x rows_in] operator: 1 to `width` taps per row (mostly not a multiple of 4), and no
    taps at all on every `empty_every`-th row."""
    counts = rng.randint(1, width + 1, size=rows_out)
    if empty_every:
        counts[1::empty_every] = 0
    rows = np.repeat(np.arange(rows_out), counts)
    cols = rng.randint(0, rows_in, size=rows.size)
    vals = rng.uniform(-1, 1, size=rows.size)
    m = sp.csr_matrix((vals, (rows, cols)), shape=(rows_out, rows_in))
    m.sum_duplicates()
    return m.astype(np.float32)


def _unpool3(rng, rows_out, rows_in):
    """An up-sampling operator: every row a barycentric combination of three source rows."""
    cols = np.stack([rng.choice(rows_in, 3, replace=False) for _ in range(rows_out)])
    w = rng.dirichlet(np.ones(3), size=rows_out)
    return sp.csr_matrix((w.ravel(), (np.repeat(np.arange(rows_out), 3), cols.ravel())),
                         shape=(rows_out, rows_in)).astype(np.float32)


def _apply(m, x):
    """float64 m @ x[n] for every sample (m None: identity)."""
    x = x.astype(np.float64)
    if m is None:
        return x
    m = m.astype(np.float64)
    return np.stack([m @ x[n] for n in range(x.shape[0])])


def _rowsum(m, rows):
    return np.ones(rows) if m is None else np.asarray(m.astype(np.float64).sum(axis=1)).ravel()


def _cheb_L0(hierarchy, K=3):
    from cape_b200 import topology as topo
    T = topo.cheb_polynomials(hierarchy["L"][0], K)
    return [None] + [t.astype(np.float32) for t in T[1:]]


def _op_id(tp, m):
    return -1 if m is None else tp.add_operator(m)


def _buffer(n, fill, head=0):
    """A flat device buffer of head + n + GUARD floats filled with `fill` (a scalar or an array of n values for the
    target); returns (device buffer, host copy of its initial contents, mask of the n target elements)."""
    init = np.full(head + n + GUARD, NAN, np.float32)
    init[head:head + n] = fill
    mask = np.zeros(init.size, bool)
    mask[head:head + n] = True
    return torch.from_numpy(init).to(_dev()), init, mask


def _pad(a, v):
    """a flattened, followed by the GUARD sentinel positions (value v)."""
    return np.concatenate([a.ravel(), np.full(GUARD, v, a.dtype)])


def _dev_view(host, off=0):
    """Device copy of a float32 array at an element offset `off` into a larger buffer (off = 1: not 16-byte aligned)."""
    buf = torch.full((host.size + off,), float("nan"), device=_dev())
    buf[off:] = torch.from_numpy(np.ascontiguousarray(host).ravel())
    return buf[off:].view(host.shape)


# ---------------------------------------------------------------------------------------------------------------------
# cape_cheb_fwd: thin input (thin_fwd_kernel) and thin output (thinout_project_kernel + thinout_combine_kernel)
# ---------------------------------------------------------------------------------------------------------------------
def conv_case(N, rows_out, ncols, terms, *, tp=None, slots=(), C=5, epilogue="linear", act="none", bias=None,
              out2=False, misalign=(), shared_src=False, seed=0):
    """terms: list of (F, m, src_stride) with m a scipy operator [rows_out x src_rows] or None (identity).
    slots: indices of the terms that carry condition weights.  bias: None | 'shared' | 'row'.
    misalign: any of 'out', 'aux', 'bias' -- that operand 4 bytes off 16-byte alignment.
    Returns (kernel names, worst relative error)."""
    E, dev = _E(), _dev()
    tp = tp or _tp()
    rng = np.random.RandomState(seed)
    act_id, alpha = ACTS[act]
    cond = rng.normal(size=(N, C)).astype(np.float32) if slots else None
    pre = np.zeros((N, rows_out, ncols))
    dterms = []
    for i, (F, m, stride) in enumerate(terms):
        src_rows = rows_out if m is None else m.shape[1]
        if not (shared_src and i):                              # shared_src: every term reads the first one's source
            src = rng.normal(size=(N, src_rows, stride)).astype(np.float32)
            src[:, :, F:] = NAN                                 # columns past F must never be read
            src_d = torch.from_numpy(src).to(dev)
        # weights and condition weights at a row stride of 2 * ncols; the interleaved rows are NaN
        wbuf = np.full((F, 2, ncols), NAN, np.float32)
        wbuf[:, 0, :] = rng.normal(0, 1 / np.sqrt(F), size=(F, ncols))
        t = dict(src=src_d, op=_op_id(tp, m), F=F, src_rows=src_rows, src_stride=stride,
                 w=torch.from_numpy(wbuf).to(dev)[:, 0, :], w_stride=2 * ncols)
        w64 = wbuf[:, 0, :].astype(np.float64)      # the narrower side first: (m . x) W == m . (x W)
        pre += _apply(m, src[:, :, :F]) @ w64 if F <= ncols else _apply(m, src[:, :, :F].astype(np.float64) @ w64)
        if i in slots:
            wcb = np.full((C, 2, ncols), NAN, np.float32)
            wcb[:, 0, :] = rng.normal(size=(C, ncols))
            t["wc"] = torch.from_numpy(wcb).to(dev)[:, 0, :]
            pre += _rowsum(m, rows_out)[None, :, None] * (cond.astype(np.float64) @ wcb[:, 0, :])[:, None, :]
        dterms.append(t)
    total = N * rows_out * ncols
    b = None
    if bias is not None:
        b = rng.normal(size=(rows_out, ncols) if bias == "row" else (ncols,)).astype(np.float32)
    aux = rng.normal(size=(N, rows_out, ncols)).astype(np.float32) if epilogue in ("slope", "dualmask") else None
    if epilogue == "linear":
        v = pre + (b.astype(np.float64) if b is not None else 0.0)
        want = [v if act == "none" else (np.maximum(v, 0) if act == "relu" else np.where(v > 0, v, alpha * v))]
    elif epilogue == "slope":
        want = [pre * np.where(aux > 0, 1.0, alpha)]
    else:
        want = [pre] + ([np.where(aux > 0, pre, 0.0)] if out2 else [])
    head = 1 if "out" in misalign else 0
    outs = [_buffer(total, NAN, head) for _ in want]
    views = [d[head:head + total].view(N, rows_out, ncols) for d, _, _ in outs]
    epi = {"linear": E.EPI_LINEAR, "slope": E.EPI_SLOPE, "dualmask": E.EPI_DUALMASK}[epilogue]
    cond_d = torch.from_numpy(cond).to(dev) if cond is not None else None
    bias_d = _dev_view(b, 1 if "bias" in misalign else 0) if b is not None else None
    aux_d = _dev_view(aux, 1 if "aux" in misalign else 0) if aux is not None else None

    def call():
        E.cheb_call(tp, N, rows_out, ncols, dterms, views[0], out2=views[1] if len(views) > 1 else None, cond=cond_d,
                    epilogue=epi, act=act_id, alpha=alpha, bias=bias_d, bias_per_row=bias == "row", aux=aux_d)

    def reset():
        for d, init, _ in outs:
            d.copy_(torch.from_numpy(init))
    names = _traced(call, reset)
    err = 0.0
    for (d, init, mask), w in zip(outs, want):
        full = np.full(init.size, np.nan)
        full[head:head + total] = w.ravel()
        err = max(err, _check(d.cpu().numpy(), init, mask, full, "cheb_fwd"))
    return names, err


def thin_fwd(case, *args, **kw):
    names, err = conv_case(*args, **kw)
    _expect(names, ["thin_fwd_kernel"], launches=1)
    _report(case, err)


def generic_fwd(case, *args, tc=True, tuning=(), **kw):
    """A call the thin kernels must reject: the generic gather kernel computes it (tensor cores on or off)."""
    with _knobs(tuning, tc=tc):
        names, err = conv_case(*args, **kw)
    _expect(names, ["ellconv_kernel"], launches=1, thin=False)
    _report(case, err)


def thinout(case, *args, **kw):
    names, err = conv_case(*args, shared_src=True, **kw)
    assert names == ["thinout_project_kernel", "thinout_combine_kernel"], names
    _report(case, err)


# ---- thin input: channels and columns (ncols 16 / 20 / 64 / 128 on the vec4 path, 18 / 33 / 127 scalar)
@pytest.mark.parametrize("ncols", [16, 20, 64, 128, 18, 33, 127])
@pytest.mark.parametrize("F", [1, 2, 3, 4])
def test_thin_fwd_channels(F, ncols):
    rng = np.random.RandomState(F * 1000 + ncols)
    m = _operator(rng, 37, 37)
    thin_fwd("thin_fwd F=%d ncols=%d" % (F, ncols), 5, 37, ncols, [(F, m, F), (F, None, F)], bias="shared",
             seed=F + ncols)


# mixed F within one call, identity and gathered terms, 1 to 8 terms, up to KF = 32
@pytest.mark.parametrize("Fs", [[3], [3, 1, 4, 2], [2, 4, 1, 3, 4], [4] * 8, [1, 2, 3, 4, 4, 4, 3, 1]])
@pytest.mark.parametrize("ncols", [64, 33])
def test_thin_fwd_terms(Fs, ncols):
    rng = np.random.RandomState(len(Fs))
    terms = [(F, None if i % 3 == 1 else _operator(rng, 129, 129, width=5 + i), F) for i, F in enumerate(Fs)]
    thin_fwd("thin_fwd Fs=%s ncols=%d" % (Fs, ncols), 3, 129, ncols, terms, slots=(0,), seed=7)


# rows_out of 5 .. 129 with total_rows % 128 != 0, and a single sample
@pytest.mark.parametrize("rows_out,N", [(5, 31), (37, 5), (127, 3), (128, 3), (129, 1), (129, 7), (300, 1)])
def test_thin_fwd_rows(rows_out, N):
    rng = np.random.RandomState(rows_out)
    terms = [(3, None, 3), (3, _operator(rng, rows_out, rows_out), 3), (3, _operator(rng, rows_out, rows_out), 3)]
    thin_fwd("thin_fwd rows_out=%d N=%d" % (rows_out, N), N, rows_out, 64, terms, bias="row", act="leaky")


# the real first-level Chebyshev operators (6890 rows, up to ~30 taps per row), as in the encoder's first conv
def test_thin_fwd_L0(hierarchy):
    ops = _cheb_L0(hierarchy)
    thin_fwd("thin_fwd L0 K=3 3->64", 3, 6890, 64, [(3, m, 3) for m in ops], bias="shared", act="leaky")


# pooling (rows_out < src_rows) and a 3-tap unpooling, F = 3 inside a 7-wide source buffer
@pytest.mark.parametrize("ncols", [32, 127])
def test_thin_fwd_pool_unpool(ncols):
    rng = np.random.RandomState(ncols)
    pool = _operator(rng, 61, 250)
    thin_fwd("thin_fwd pool ncols=%d" % ncols, 3, 61, ncols, [(3, pool, 7), (2, _operator(rng, 61, 250), 2)])
    up = _unpool3(rng, 250, 61)
    thin_fwd("thin_fwd unpool ncols=%d" % ncols, 3, 250, ncols, [(3, up, 7), (1, None, 1)], slots=(0,))


# condition slots: tiles that span up to 27 samples, C of 5 and 72, one to three slots; (21, 128) and (9, 32 x 2 slots)
# fill the condition staging buffer exactly (max_samples * nslots * ncols = 1024)
@pytest.mark.parametrize("rows_out,ncols,C,nslots", [(5, 16, 5, 1), (5, 16, 72, 2), (37, 64, 72, 3), (21, 128, 5, 1),
                                                     (9, 32, 72, 2), (128, 100, 5, 2)])
def test_thin_fwd_condition(rows_out, ncols, C, nslots):
    rng = np.random.RandomState(rows_out + ncols)
    terms = [(3, None, 3), (3, _operator(rng, rows_out, rows_out), 3), (2, _operator(rng, rows_out, rows_out), 5)]
    thin_fwd("thin_fwd cond rows_out=%d ncols=%d C=%d slots=%d" % (rows_out, ncols, C, nslots), 60, rows_out, ncols,
             terms, slots=tuple(range(3 - nslots, 3)), C=C, bias="shared")


# one past the staging buffer (1152 and 1088 > 1024): the call falls back to the generic kernel and is still right
@pytest.mark.parametrize("tc", [True, False])
@pytest.mark.parametrize("rows_out,ncols,C,nslots", [(18, 128, 5, 1), (8, 32, 72, 2)])
def test_thin_fwd_condition_over(rows_out, ncols, C, nslots, tc):
    rng = np.random.RandomState(rows_out)
    terms = [(3, None, 3), (3, _operator(rng, rows_out, rows_out), 3)]
    generic_fwd("thin_fwd cond over rows_out=%d ncols=%d tc=%d" % (rows_out, ncols, tc), 40, rows_out, ncols, terms,
                slots=tuple(range(nslots)), C=C, tc=tc)


# LINEAR: no / shared / per-row bias, each with no activation, leaky (alpha 0.2 and 0.37) and ReLU, vec4 and scalar
@pytest.mark.parametrize("act", ["none", "leaky", "leaky.37", "relu"])
@pytest.mark.parametrize("bias", [None, "shared", "row"])
@pytest.mark.parametrize("ncols", [64, 33])
def test_thin_fwd_linear(ncols, bias, act):
    rng = np.random.RandomState(3)
    terms = [(3, None, 3), (3, _operator(rng, 100, 100), 3)]
    thin_fwd("thin_fwd linear ncols=%d bias=%s act=%s" % (ncols, bias, act), 3, 100, ncols, terms, bias=bias, act=act)


# SLOPE, DUALMASK with and without out2 (data gradients of a leaky-ReLU layer), vec4 and scalar
@pytest.mark.parametrize("epilogue,out2,act", [("slope", False, "leaky"), ("slope", False, "leaky.37"),
                                               ("dualmask", True, "none"), ("dualmask", False, "none")])
@pytest.mark.parametrize("ncols", [64, 33])
def test_thin_fwd_epilogues(ncols, epilogue, out2, act):
    rng = np.random.RandomState(4)
    terms = [(1, _operator(rng, 100, 100), 1), (1, None, 1)]
    thin_fwd("thin_fwd %s out2=%d alpha=%s ncols=%d" % (epilogue, out2, ACTS[act][1], ncols), 3, 100, ncols, terms,
             epilogue=epilogue, act=act, out2=out2)


# ncols % 4 == 0 but out, aux or bias off 16-byte alignment: the scalar column path
@pytest.mark.parametrize("which,epilogue,bias", [("out", "linear", "row"), ("bias", "linear", "shared"),
                                                 ("aux", "dualmask", None), ("out", "slope", None)])
def test_thin_fwd_misaligned(which, epilogue, bias):
    rng = np.random.RandomState(5)
    terms = [(4, _operator(rng, 90, 90), 4), (2, None, 2)]
    thin_fwd("thin_fwd misaligned %s %s" % (which, epilogue), 3, 90, 64, terms, epilogue=epilogue, bias=bias,
             out2=epilogue == "dualmask", misalign=(which,), act="leaky" if epilogue != "dualmask" else "none")


# ---- thin output: ncols 1..4, F of 32 .. 512 (the project kernel's 8 / 16 / 32 lanes per row and their tails)
@pytest.mark.parametrize("F", [32, 36, 60, 64, 100, 128, 132, 512])
@pytest.mark.parametrize("ncols", [1, 2, 3, 4])
def test_thinout_shapes(ncols, F):
    rng = np.random.RandomState(F + ncols)
    nterms = 1 + (F // 4 + ncols) % 4
    stride = F + 4 * (ncols % 2)
    ms = [None] + [_operator(rng, 211, 211, width=3 + 4 * i) for i in range(nterms - 1)]
    thinout("thinout ncols=%d F=%d terms=%d stride=%d" % (ncols, F, nterms, stride), 3, 211, ncols,
            [(F, m, stride) for m in ms], bias="shared")


# pooled (rows_out < src_rows) and 3-tap unpooled operators, src_stride > F
@pytest.mark.parametrize("ncols", [1, 3])
def test_thinout_pool_unpool(ncols):
    rng = np.random.RandomState(ncols)
    pool = [_operator(rng, 90, 301) for _ in range(2)]
    thinout("thinout pool ncols=%d" % ncols, 4, 90, ncols, [(64, m, 72) for m in pool], act="leaky")
    up = [_unpool3(rng, 301, 90)] + [_operator(rng, 301, 90) for _ in range(3)]
    thinout("thinout unpool ncols=%d" % ncols, 4, 301, ncols, [(36, m, 40) for m in up], bias="row")


# 64 samples of the first level: the project kernel's grid-stride loop wraps ~13 times
@pytest.mark.parametrize("F", [36, 132])
def test_thinout_grid_wrap(hierarchy, F):
    ops = _cheb_L0(hierarchy)
    thinout("thinout L0 N=64 F=%d" % F, 64, 6890, 3, [(F, m, F) for m in ops], bias="row")


# condition slots: up to four, rows_out 37 (a 256-row block touches at most 255 // 37 + 2 = 8 samples, the limit) .. 300
@pytest.mark.parametrize("rows_out,nslots,C", [(37, 1, 5), (37, 4, 72), (43, 2, 5), (42, 3, 72), (300, 4, 5)])
def test_thinout_condition(rows_out, nslots, C):
    rng = np.random.RandomState(rows_out)
    ms = [None] + [_operator(rng, rows_out, rows_out) for _ in range(3)]
    thinout("thinout cond rows_out=%d slots=%d C=%d" % (rows_out, nslots, C), 50, rows_out, 3,
            [(32, m, 32) for m in ms], slots=tuple(range(nslots)), C=C, bias="shared")


@pytest.mark.parametrize("act", ["none", "leaky", "relu"])
@pytest.mark.parametrize("bias", [None, "shared", "row"])
def test_thinout_bias_act(bias, act):
    rng = np.random.RandomState(9)
    ms = [None, _operator(rng, 150, 150)]
    thinout("thinout bias=%s act=%s" % (bias, act), 3, 150, 4, [(64, m, 64) for m in ms], bias=bias, act=act)


# calls the thin-output kernels reject: knob 7, a workspace smaller than z, 5 terms, F of 516 / 30 / 34, ncols = 5,
# and rows_out = 36 with condition slots (255 // 36 + 2 = 9 samples per block)
@pytest.mark.parametrize("tc", [True, False])
@pytest.mark.parametrize("why", ["knob7", "workspace", "5terms", "F516", "F30", "F34", "ncols5", "rows36"])
def test_thinout_fallback(why, tc):
    rng = np.random.RandomState(11)
    N, rows, ncols, F, nterms, kw = 3, 120, 3, 64, 3, {}
    tuning = ((7, 1),) if why == "knob7" else ()
    if why == "5terms":
        nterms = 5
    elif why.startswith("F"):
        F = int(why[1:])
    elif why == "ncols5":
        ncols = 5
    elif why == "rows36":
        N, rows, kw = 20, 36, dict(slots=(0, 1), C=5)
    elif why == "workspace":
        tp = _E().Topology(0)
        tp.reserve_workspace(N * rows * 16 * 4 - 16)      # z needs N * src_rows * 16 floats
        kw["tp"] = tp
    ms = [None] + [_operator(rng, rows, rows) for _ in range(nterms - 1)]
    generic_fwd("thinout fallback %s tc=%d" % (why, tc), N, rows, ncols, [(F, m, F) for m in ms], shared_src=True,
                bias="shared", tc=tc, tuning=tuning, **kw)


# ---------------------------------------------------------------------------------------------------------------------
# cape_cheb_dw with F <= 4: thin_dw_kernel<KF> + reduce_splits_kernel
# ---------------------------------------------------------------------------------------------------------------------
def dw_case(N, rows_out, ncols, F, ms, *, tp=None, single=False, src_rows=None, src_stride=None, accumulate=False,
            g_off=0, seed=0):
    """dW_j (+)= sum_n (m_j . src[n][:, :F])^T . g[n] for every operator m_j (None: identity), written into terms
    1 .. nops of a [F, nops + 2, ncols + 4] buffer (dw_stride = (nops + 2) * (ncols + 4), dw_term_stride = ncols + 4):
    the terms before and after and the four columns after every row are sentinels.  single: the nops = 0 form
    (one operator).  g_off = 1: g off 16-byte alignment.  Returns (kernel names, relative error)."""
    E, dev = _E(), _dev()
    tp = tp or _tp()
    rng = np.random.RandomState(seed)
    src_rows = src_rows or rows_out
    src_stride = src_stride or F
    nops = len(ms)
    src = rng.normal(size=(N, src_rows, src_stride)).astype(np.float32)
    src[:, :, F:] = NAN
    g = rng.normal(size=(N, rows_out, ncols)).astype(np.float32)
    K, W = nops + 2, ncols + 4
    init = (rng.normal(size=(F, K, W)) if accumulate else np.full((F, K, W), np.nan)).astype(np.float32)
    want = init.astype(np.float64)
    for j, m in enumerate(ms):
        d = np.einsum("nrf,nrc->fc", _apply(m, src[:, :, :F]), g.astype(np.float64))
        want[:, 1 + j, :ncols] = want[:, 1 + j, :ncols] + d if accumulate else d
    mask = np.zeros((F, K, W), bool)
    mask[:, 1:1 + nops, :ncols] = True
    buf = torch.from_numpy(np.concatenate([init.ravel(), np.full(GUARD, NAN, np.float32)])).to(dev)
    ids = [_op_id(tp, m) for m in ms]
    src_d, g_d = torch.from_numpy(src).to(dev), _dev_view(g, g_off)
    dw = buf[W:]                                            # term 1

    def call():
        if single:
            E.cheb_dw(tp, N, rows_out, ncols, src_d, ids[0], F, src_rows, src_stride, g_d, dw, K * W,
                      accumulate=accumulate)
        else:
            E.cheb_dw(tp, N, rows_out, ncols, src_d, ids, F, src_rows, src_stride, g_d, dw, K * W,
                      accumulate=accumulate, dw_term_stride=W)
    names = _traced(call, lambda: buf.copy_(torch.from_numpy(_pad(init, NAN))))
    err = _check(buf.cpu().numpy(), _pad(init, NAN), _pad(mask, False), _pad(want, np.nan), "cheb_dw")
    return names, err


def _template(nq):
    return 4 if nq <= 4 else (8 if nq <= 8 else (12 if nq <= 12 else 16))


def thin_dw(case, *args, **kw):
    names, err = dw_case(*args, **kw)
    nops = 1 if kw.get("single") else len(args[4])
    _expect(names, ["thin_dw_kernel<%d>" % _template(nops * args[3]), "reduce_splits_kernel"], launches=2)
    _report(case, err)


def generic_dw(case, *args, tc=True, **kw):
    with _knobs(tc=tc):
        names, err = dw_case(*args, **kw)
    _expect(names, ["ellconv_dw_kernel"], thin=False)
    _report(case, err)


# both ends of every template: nops * F of 1 and 4 (<4>), 6 and 8 (<8>), 9 and 12 (<12>), 16 (<16>); nops * F of 5 or
# 13 cannot be formed with nops <= 4 and F <= 4
@pytest.mark.parametrize("ncols", [32, 64, 128, 256])
@pytest.mark.parametrize("nops,F", [(1, 1), (1, 4), (4, 1), (2, 3), (3, 2), (2, 4), (3, 3), (4, 3), (3, 4), (4, 4)])
def test_thin_dw_templates(nops, F, ncols):
    rng = np.random.RandomState(nops * 10 + F)
    ms = [None] + [_operator(rng, 333, 333, width=4 + 3 * j) for j in range(nops - 1)]
    thin_dw("thin_dw nops=%d F=%d ncols=%d" % (nops, F, ncols), 3, 333, ncols, F, ms, seed=ncols)


# the single-term form (nops = 0), overwrite and accumulate
@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("F,ncols", [(1, 32), (3, 256), (4, 64)])
def test_thin_dw_single(F, ncols, accumulate):
    rng = np.random.RandomState(F)
    thin_dw("thin_dw single F=%d ncols=%d acc=%d" % (F, ncols, accumulate), 4, 500, ncols, F,
            [_operator(rng, 500, 700)], single=True, src_rows=700, src_stride=F + 3, accumulate=accumulate)


# accumulation into the strided multi-term slice; a pooled source with src_stride > F
@pytest.mark.parametrize("ncols", [64, 256])
def test_thin_dw_accumulate_strided(ncols):
    rng = np.random.RandomState(ncols)
    ms = [_operator(rng, 400, 650) for _ in range(3)]
    thin_dw("thin_dw acc pool ncols=%d" % ncols, 3, 400, ncols, 3, ms, src_rows=650, src_stride=7, accumulate=True)


# total_rows < 256, total_rows % 256 != 0, and 64 samples of the first level (441k rows)
@pytest.mark.parametrize("N,rows", [(1, 200), (3, 1001), (1, 5)])
def test_thin_dw_rows(N, rows):
    rng = np.random.RandomState(rows)
    ms = [None, _operator(rng, rows, rows), _operator(rng, rows, rows)]
    thin_dw("thin_dw N=%d rows=%d" % (N, rows), N, rows, 128, 3, ms)


def test_thin_dw_L0(hierarchy):
    thin_dw("thin_dw L0 N=64 K=3 F=3 ncols=64", 64, 6890, 64, 3, _cheb_L0(hierarchy), accumulate=True)


# the operand swap of a thin-OUTPUT layer's weight gradient, exactly as CapeNetwork calls it: the operators' transposes
# on the narrow gradient g [N, rows_out, Fout], one pass over the wide input x [N, rows_in, F], dW in the [F, K, Fout]
# layout through dw_stride = 1, dw_term_stride = Fout, dw_col_stride = K * Fout
@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("F,Fout,K", [(32, 1, 3), (64, 3, 3), (128, 3, 2), (256, 4, 4), (64, 2, 1)])
def test_thin_dw_swap(F, Fout, K, accumulate):
    E, dev = _E(), _dev()
    tp = _tp()
    rng = np.random.RandomState(F + Fout)
    N, rows_in, rows_out = 3, 401, 401
    ms = [None] + [_operator(rng, rows_out, rows_in) for _ in range(K - 1)]
    opsT = [-1 if m is None else tp.add_operator(sp.csr_matrix(m.T)) for m in ms]
    x = rng.normal(size=(N, rows_in, F)).astype(np.float32)
    g = rng.normal(size=(N, rows_out, Fout)).astype(np.float32)
    head = 5
    init = np.full(head + F * K * Fout + GUARD, NAN, np.float32)
    if accumulate:
        init[head:head + F * K * Fout] = rng.normal(size=F * K * Fout)
    want3 = init[head:head + F * K * Fout].astype(np.float64).reshape(F, K, Fout)
    for k, m in enumerate(ms):
        H = _apply(None if m is None else sp.csr_matrix(m.T), g)          # op_k^T g: [N, rows_in, Fout]
        d = np.einsum("nrf,nrc->fc", x.astype(np.float64), H)
        want3[:, k, :] = want3[:, k, :] + d if accumulate else d
    want = np.full(init.size, np.nan)
    want[head:head + F * K * Fout] = want3.ravel()
    mask = np.zeros(init.size, bool)
    mask[head:head + F * K * Fout] = True
    buf = torch.from_numpy(init).to(dev)
    g_d, x_d = torch.from_numpy(g).to(dev), torch.from_numpy(x).to(dev)

    def call():
        E.cheb_dw(tp, N, rows_in, F, g_d, opsT, Fout, rows_out, Fout, x_d, buf[head:], 1, accumulate=accumulate,
                  dw_term_stride=Fout, dw_col_stride=K * Fout)
    names = _traced(call, lambda: buf.copy_(torch.from_numpy(init)))
    _expect(names, ["thin_dw_kernel<%d>" % _template(K * Fout), "reduce_splits_kernel"], launches=2)
    _report("thin_dw swap F=%d Fout=%d K=%d acc=%d" % (F, Fout, K, accumulate),
            _check(buf.cpu().numpy(), init, mask, want, "cheb_dw swap"))


# block counts: limited by the workspace (a fresh topology with room for 3 or 1 blocks' partials, so each block walks
# many 256-row chunks), and knob 17 (4 blocks per SM instead of the register-limited wave)
@pytest.mark.parametrize("blocks", [3, 1])
def test_thin_dw_workspace_limited(blocks):
    E = _E()
    tp = E.Topology(0)
    nops, F, ncols = 3, 4, 64
    tp.reserve_workspace(blocks * nops * F * ncols * 4)
    rng = np.random.RandomState(blocks)
    ms = [None] + [_operator(rng, 2000, 2000) for _ in range(nops - 1)]
    thin_dw("thin_dw workspace %d blocks" % blocks, 8, 2000, ncols, F, ms, tp=tp, seed=blocks)


def test_thin_dw_knob17():
    rng = np.random.RandomState(17)
    ms = [None] + [_operator(rng, 6890, 6890) for _ in range(3)]
    with _knobs(((17, 1),)):
        thin_dw("thin_dw knob17 N=20", 20, 6890, 32, 3, ms)


# calls thin_dw rejects: no workspace, ncols = 48, g off 16-byte alignment, F = 5 -- each computed by the generic
# weight-gradient kernel, in the single and the multi-term form, tensor cores on and off
@pytest.mark.parametrize("tc", [True, False])
@pytest.mark.parametrize("single", [True, False])
@pytest.mark.parametrize("why", ["no-workspace", "ncols48", "misaligned-g", "F5"])
def test_thin_dw_fallback(why, single, tc):
    rng = np.random.RandomState(21)
    ncols, F, kw = 64, 3, {}
    if why == "no-workspace":
        kw["tp"] = _E().Topology(0)
    elif why == "ncols48":
        ncols = 48
    elif why == "misaligned-g":
        kw["g_off"] = 1
    else:
        F = 5
    ms = [_operator(rng, 700, 700)] + ([] if single else [None, _operator(rng, 700, 700)])
    generic_dw("thin_dw fallback %s single=%d tc=%d" % (why, single, tc), 3, 700, ncols, F, ms, single=single,
               accumulate=not single, tc=tc, **kw)


# ---------------------------------------------------------------------------------------------------------------------
# glue kernels
# ---------------------------------------------------------------------------------------------------------------------
# cape_colsum: out[n, j, :] += sum_r coef_j[r] g[n, r, :], coef_j = rowsum of operator j (None: ones); vec path at
# ncols 4 / 8 / 64 / 512, scalar at 3 / 12 / 516; rows < 64, rows that leave a tail after the 4-row unroll, N > 4 x SMs
@pytest.mark.parametrize("N,rows,ncols,nops,g_stride", [
    (2, 1000, 64, 1, 64), (3, 777, 4, 2, 4), (2, 40, 8, 3, 12), (2, 1500, 512, 4, 516), (600, 3001, 4, 2, 4),
    (600, 1001, 12, 2, 12), (3, 999, 3, 4, 5), (2, 333, 12, 1, 16), (2, 203, 516, 3, 520), (5, 63, 64, 2, 68)])
@pytest.mark.parametrize("prefill", [False, True])
def test_colsum(N, rows, ncols, nops, g_stride, prefill):
    E, dev = _E(), _dev()
    tp = _tp()
    if N > 4 * _sms():
        assert (4 * _sms() + N - 1) // N == 1
    rng = np.random.RandomState(rows + ncols)
    ms = [None if j % 2 else _operator(rng, rows, 50) for j in range(nops)]
    g = np.full((N, rows, g_stride), NAN, np.float32)
    g[:, :, :ncols] = rng.normal(size=(N, rows, ncols))
    out0 = rng.normal(size=(N, nops, ncols)).astype(np.float32) if prefill else np.zeros((N, nops, ncols), np.float32)
    want = out0.astype(np.float64)
    for j, m in enumerate(ms):
        want[:, j, :] += np.einsum("r,nrc->nc", _rowsum(m, rows), g[:, :, :ncols].astype(np.float64))
    d, init, mask = _buffer(out0.size, out0.ravel())
    ids = [_op_id(tp, m) for m in ms]
    g_d = torch.from_numpy(g).to(dev)
    names = _traced(lambda: E.colsum(tp, g_d, N, rows, ncols, ids, d, g_stride=g_stride),
                    lambda: d.copy_(torch.from_numpy(init)))
    _expect(names, ["colsum_kernel"], launches=1)
    full = _pad(want, np.nan)
    _report("colsum N=%d rows=%d ncols=%d nops=%d gs=%d prefill=%d" % (N, rows, ncols, nops, g_stride, prefill),
            _check(d.cpu().numpy(), init, mask, full, "colsum"))


# cape_resample with a condition (fit_cond_dim + concat + unpool): y[n, r, :F] = op . x[n], y[n, r, F:F+C] =
# rowsum(op)[r] cond[n]; pool / unpool / identity, vec (F % 4 == 0) and scalar paths, C > 32, y_stride > F + C
@pytest.mark.parametrize("kind", ["pool", "unpool", "identity"])
@pytest.mark.parametrize("F,C,y_stride,x_stride", [(64, 8, 72, 64), (64, 72, 140, 68), (13, 5, 21, 13),
                                                   (13, 72, 90, 15), (3, 40, 43, 3)])
def test_resample_cond(kind, F, C, y_stride, x_stride):
    E, dev = _E(), _dev()
    tp = _tp()
    rng = np.random.RandomState(F + C)
    N = 3
    if kind == "pool":
        m, rows_out, rows_in = _operator(rng, 97, 390), 97, 390
    elif kind == "unpool":
        m, rows_out, rows_in = _unpool3(rng, 390, 97), 390, 97
    else:
        m, rows_out, rows_in = None, 211, 211
    x = np.full((N, rows_in, x_stride), NAN, np.float32)
    x[:, :, :F] = rng.normal(size=(N, rows_in, F))
    cond = rng.normal(size=(N, C)).astype(np.float32)
    want = np.full((N, rows_out, y_stride), np.nan)
    want[:, :, :F] = _apply(m, x[:, :, :F])
    want[:, :, F:F + C] = _rowsum(m, rows_out)[None, :, None] * cond.astype(np.float64)[:, None, :]
    mask = np.zeros((N, rows_out, y_stride), bool)
    mask[:, :, :F + C] = True
    d, init, _ = _buffer(want.size, NAN)
    op = _op_id(tp, m)
    x_d, c_d = torch.from_numpy(x).to(dev), torch.from_numpy(cond).to(dev)
    names = _traced(lambda: E.resample(tp, op, x_d, d, N, rows_out, rows_in, F, x_stride=x_stride, y_stride=y_stride,
                                       cond=c_d), lambda: d.copy_(torch.from_numpy(init)))
    _expect(names, ["resample_kernel"], launches=1)
    _report("resample %s F=%d C=%d ys=%d xs=%d" % (kind, F, C, y_stride, x_stride),
            _check(d.cpu().numpy(), init, _pad(mask, False), _pad(want, np.nan), "resample"))


# cape_gemm_batch through SmallGemmBatch: items with M, N, K of 1 / 63 / 65 / 130, transposed operands (a_rs == 1),
# alpha != 1, several beta = 1 items adding into one C, outputs inside wider buffers; then the same device table
# relaunched after the operands change in place (how the step reuses its tables under CUDA graphs)
def test_gemm_batch():
    E, dev = _E(), _dev()
    tp = _tp()
    rng = np.random.RandomState(0)
    # (M, N, K, transpose A, transpose B, alpha, beta, output id); outputs 7 and 8 take several beta = 1 items each
    spec = [(1, 1, 1, False, False, 1.0, 0, 0), (63, 65, 130, True, False, 0.5, 0, 1),
            (130, 63, 65, False, True, -1.5, 0, 2), (65, 130, 63, True, True, 1.0, 0, 3),
            (1, 130, 65, False, False, 2.0, 0, 4), (130, 1, 63, True, False, 1.0, 0, 5),
            (63, 63, 1, False, False, 1.0, 0, 6),
            (65, 63, 130, False, False, 1.0, 1, 7), (65, 63, 1, True, False, 0.25, 1, 7),
            (65, 63, 63, False, True, -1.0, 1, 7),
            (1, 65, 130, True, True, 1.0, 1, 8), (1, 65, 63, False, False, 3.0, 1, 8)]
    outs = {}
    for (M, N, K, ta, tb, alpha, beta, o) in spec:
        outs.setdefault(o, (M, N, beta))
    # every output is the left [M, N] block of an [M, N + 3] buffer followed by GUARD sentinels
    bufs, inits, masks = {}, {}, {}
    for o, (M, N, beta) in outs.items():
        init = np.full(M * (N + 3) + GUARD, NAN, np.float32)
        mask = np.zeros(init.size, bool)
        mask[:M * (N + 3)].reshape(M, N + 3)[:, :N] = True
        bufs[o], inits[o], masks[o] = torch.from_numpy(init).to(dev), init, mask
    ops = []
    for (M, N, K, ta, tb, alpha, beta, o) in spec:
        A = torch.empty(K, M, device=dev).t() if ta else torch.empty(M, K, device=dev)
        B = torch.empty(N, K, device=dev).t() if tb else torch.empty(K, N, device=dev)
        Cv = bufs[o][:M * (N + 3)].view(M, N + 3)[:, :N]
        ops.append((A, B, Cv, alpha, beta, o))
    batch = E.SmallGemmBatch(tp)
    for trip in range(2):
        want = {}
        for o, (M, N, beta) in outs.items():
            init = inits[o].copy()
            if beta:                                      # accumulating outputs start from known values
                init[masks[o]] = rng.normal(size=int(masks[o].sum()))
            bufs[o].copy_(torch.from_numpy(init))
            inits[o] = init
            want[o] = init.astype(np.float64)
        for (A, B, Cv, alpha, beta, o), (M, N, K, *_) in zip(ops, spec):
            a, b = rng.normal(size=(M, K)).astype(np.float32), rng.normal(size=(K, N)).astype(np.float32)
            A.copy_(torch.from_numpy(a))                  # in place: the table keeps the same pointers
            B.copy_(torch.from_numpy(b))
            prod = alpha * (a.astype(np.float64) @ b.astype(np.float64))
            w = want[o][:M * (N + 3)].reshape(M, N + 3)
            w[:, :N] = w[:, :N] + prod if beta else prod

        def launch():
            for A, B, Cv, alpha, beta, _ in ops:
                batch.add(A, B, Cv, alpha=alpha, beta=beta)
            batch.flush()

        def reset():
            for o in outs:
                bufs[o].copy_(torch.from_numpy(inits[o]))
        names = _traced(launch, reset)
        assert len(batch.tables) == 1, "the second flush must reuse the first one's device table"
        _expect(names, ["gemm_batch_kernel"], launches=1)
        for o in outs:
            _report("gemm_batch trip %d output %d" % (trip, o),
                    _check(bufs[o].cpu().numpy(), inits[o], masks[o], np.where(masks[o], want[o], np.nan),
                           "gemm_batch output %d" % o))
