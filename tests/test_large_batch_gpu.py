"""The training step at batch 256, four times the benchmarked batch, against the fp32 oracle.

The batch changes which kernels run, not only how many rows they take: the weight-gradient kernels' row splits grow
with it (their split plan keeps the number of CTAs fixed), and the thin-output projection of `dec/outputs` needs
N x 6890 x 16 floats of workspace, more than the network's 64 MB from batch 153 on, so from there that forward runs
on the generic kernels.  test_kernel_census prints, per launch tag, the kernels one forward/backward launches at batch
64 and 256, and the tags where they differ.

Each batch-256 update runs the fp32 CPU oracle: 2 to 4 minutes on 8 cores, and 35 GB (NZ64_AFFINE) to more than
60 GB (NZ18_PLAIN) of host memory.  On the device a batch-256 update peaks at 24 GB (NZ64_AFFINE) and 64 GB
(NZ18_PLAIN) on an 80 GB H100, so the two do not fit side by side; and a dropped
CapeNetwork (its layers point back at it) keeps its device buffers until Python's cyclic collector runs: each test
here starts and ends with a collection, so no network of an earlier test is still holding memory."""
import collections
import gc

import pytest
import torch

import parity
import test_gpu_thin_paths as TP

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _no_dropped_networks():
    def release():
        gc.collect()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    release()
    yield
    release()


def _cfg(name):
    from cape_b200 import params
    return dict(getattr(params, name), decay_steps=10)


@pytest.mark.parametrize("name", ["NZ64_AFFINE", "NZ18_PLAIN"])
def test_train_step_batch_256(hierarchy, name):
    """x_hat, the loss terms, every gradient and every post-update parameter of one update (the reference's
    initialisers, replayed from the captured CUDA graphs) within parity.TOL of the oracle."""
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    res = parity.train_step(hierarchy, _cfg(name), N=256, use_graph=True, fc_scale=1.0)
    print("%s batch 256: %d values, worst %s; device memory %.1f GB before, peak %.1f GB" % (
        name, len(res), max(res.items(), key=lambda kv: kv[1]), before / 1e9, torch.cuda.max_memory_allocated() / 1e9))
    bad = {k: v for k, v in res.items() if not v < parity.TOL}
    assert not bad, "parity failures (rel err): %s" % bad


def census(net):
    """{launch tag: short names of the library kernels it launches} of one forward/backward of `net`, read from the
    kernel nodes of a CUDA graph captured from it (never replayed), in launch order; launches outside any tag are under
    '(untagged)'.  Every launch the library counts is attributed to exactly one tag."""
    from cape_b200 import engine as E
    lib = TP._lib()
    spans, depth = [], [0]

    class Span:                                   # stands in for engine._Prof: the launch counter around each call
        def __init__(self, family, tag):
            self.tag = tag[0] if tag is not None else None

        def __enter__(self):
            depth[0] += 1
            self.n0 = lib.cape_launch_count()
            return self

        def __exit__(self, *exc):
            depth[0] -= 1
            if depth[0] == 0 and self.tag is not None:          # a tagged call inside another belongs to the outer one
                spans.append((self.tag, self.n0, lib.cape_launch_count()))
            return False

    prof = E._Prof
    E._Prof = Span
    try:
        with net._no_collector():
            n0 = lib.cape_launch_count()
            names = TP._captured(net.enqueue_fwd_bwd)
            n1 = lib.cape_launch_count()
    finally:
        E._Prof = prof
    assert len(names) == n1 - n0, "captured %d kernels, %d launches counted" % (len(names), n1 - n0)
    out, seen = collections.OrderedDict(), set()
    for tag, a, b in spans:
        out.setdefault(tag, []).extend(names[a - n0:b - n0])
        seen.update(range(a - n0, b - n0))
    rest = [n for i, n in enumerate(names) if i not in seen]
    if rest:
        out["(untagged)"] = rest
    assert sum(len(v) for v in out.values()) == len(names)
    return out


def _fmt(names):
    return ", ".join("%s x%d" % (k, v) if v > 1 else k for k, v in collections.Counter(names).items())


@pytest.mark.parametrize("name", ["NZ64_AFFINE", "NZ18_PLAIN"])
def test_kernel_census(hierarchy, name):
    """The kernels of every launch tag at batch 64 and 256.  `dec/outputs:fwd` cannot run the thin-output projection
    at 256 (its workspace rule); the affine model's runs it at 64."""
    from cape_b200.network import CapeNetwork
    from cape_b200.synthetic import make_batch
    h, cfg = hierarchy, _cfg(name)
    got = {}
    for N in (64, 256):
        net = CapeNetwork(h["L"], h["D"], h["U"], h["L_d"], h["D_d"], cfg, N)
        tb = {k: torch.from_numpy(v) for k, v in make_batch(N, cfg["nz"], seed=1).items()}
        net.set_inputs(tb["x_g"], tb["cond_g"], tb["cond2_g"], tb["eps"], tb["x_d"], tb["cond_d"], tb["cond2_d"])
        net.train_step(update=False)                # lazy set-up and workspace growth before the capture
        torch.cuda.synchronize()
        got[N] = census(net)
        del net
        gc.collect()                                # the network is in reference cycles
        torch.cuda.synchronize()
    print("\n%s: kernels per launch tag, batch 64" % name)
    for tag, names in got[64].items():
        print("  %-32s %s" % (tag, _fmt(names)))
    print("%s: tags whose kernels differ at batch 256" % name)
    for tag in list(got[64]) + [t for t in got[256] if t not in got[64]]:
        a, b = got[64].get(tag, []), got[256].get(tag, [])
        if a != b:
            print("  %-32s 64: %s\n  %-32s 256: %s" % (tag, _fmt(a), "", _fmt(b)))
    out64, out256 = got[64]["dec/outputs:fwd"], got[256]["dec/outputs:fwd"]
    assert not TP._ran(out256, "thinout_project_kernel"), out256
    assert name != "NZ64_AFFINE" or TP._ran(out64, "thinout_project_kernel"), out64
