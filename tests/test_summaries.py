"""TensorBoard summaries on the host: the event-file writer, the histogram limits and encoding, the histogram inventory,
the scalar tags and the moving-average recurrence (tests/summary_oracle.py holds the transcriptions they are checked
against).  The GPU side is tests/test_zzzzz_summaries_gpu.py."""
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

import summary_oracle as SO  # noqa: E402
from cape_b200 import summary as S  # noqa: E402


def _histogram_of(values):
    """(stats, counts) as cape_histogram returns them, computed on the host in float64."""
    lim = S.bucket_limits()
    x = np.asarray(values, np.float32).astype(np.float64).reshape(-1)
    counts = np.bincount(np.searchsorted(lim, x, side="right"), minlength=len(lim)).astype(np.int64)
    stats = np.array([x.min(), x.max(), x.size, x.sum(), (x * x).sum()], np.float64)
    return stats, counts


def _edge_values():
    lim = S.bucket_limits()
    inner = lim[(np.abs(lim) > 0) & (np.abs(lim) < 1e20)]
    f = inner.astype(np.float32)
    near = np.concatenate([f, np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(-np.inf))])
    return np.concatenate([near, np.float32([0.0, -0.0, 1e-13, -1e-13, 1e-45, -1e-45, 1e-39, 3e20, -3e20, 3.4e38,
                                             -3.4e38])])


def test_bucket_limits_are_tfs_table():
    lim = S.bucket_limits()
    tf = SO.TFHistogram().limits
    assert len(lim) == len(tf) == 1551
    assert lim.tolist() == tf                       # bit for bit
    assert lim[0] == -sys.float_info.max and lim[-1] == sys.float_info.max
    assert lim[775] == 0.0 and lim[776] == 1e-12 and lim[774] == -1e-12
    assert np.all(np.diff(lim) > 0)
    assert lim[-2] < 1e20 <= lim[-2] * 1.1


@pytest.mark.parametrize("kind", ["normal", "edge", "single", "sparse"])
def test_encoding_matches_tf(kind):
    """encode_histogram of host counts == TF's Histogram::Add + EncodeToProto, collapsed empty runs included."""
    from cape_b200.tf_checkpoint import _parse_proto
    rng = np.random.RandomState(3)
    values = {"normal": rng.normal(0, 0.1, 3000), "edge": _edge_values(), "single": np.float32([0.25]),
              "sparse": np.float32([-5.0, 1e-3, 1e-3, 7e4])}[kind].astype(np.float32)
    stats, counts = _histogram_of(values)
    p = _parse_proto(S.encode_histogram(stats, counts, S.bucket_limits()))
    f64 = lambda b: np.frombuffer(b, "<f8")
    mn, mx, num, sm, sq, lim, cnt = SO.tf_histogram(values).encode()
    assert f64(p[1][0])[0] == mn and f64(p[2][0])[0] == mx and f64(p[3][0])[0] == num
    assert abs(f64(p[4][0])[0] - sm) <= 1e-12 * np.abs(values.astype(np.float64)).sum()
    assert abs(f64(p[5][0])[0] - sq) <= 1e-12 * sq
    assert f64(p[6][0]).tolist() == lim
    assert f64(p[7][0]).tolist() == cnt


def test_writer_round_trip(tmp_path):
    w = S.EventWriter(str(tmp_path))
    name = os.path.basename(w.path)
    assert name.startswith("events.out.tfevents.") and len(name.split(".")[3]) == 10
    vals = np.random.RandomState(0).normal(size=500).astype(np.float32)
    stats, counts = _histogram_of(vals)
    scalars = list(zip(S.SCALAR_TAGS, np.linspace(-1, 1, len(S.SCALAR_TAGS))))
    histo = S.encode_histogram(stats, counts, S.bucket_limits())
    w.add(7, scalars, [("a/weights", histo)])
    w.add(9, [("validation/loss", 1.5)])
    # flushed after every event: readable before close
    ev = SO.read_events(w.path)
    w.close()
    assert len(ev) == 3 and ev[0]["file_version"] == "brain.Event:2"
    assert [e["step"] for e in ev[1:]] == [7, 9]
    assert ev[1]["tags"] == list(S.SCALAR_TAGS) + ["a/weights"]
    for t, v in scalars:
        assert ev[1]["scalars"][t] == np.float32(v)
    h = ev[1]["histograms"]["a/weights"]
    mn, mx, num, sm, sq, lim, cnt = SO.tf_histogram(vals).encode()
    assert (h["min"], h["max"], h["num"]) == (mn, mx, num)
    assert h["bucket_limit"] == lim and h["bucket"] == cnt
    assert ev[2]["scalars"] == {"validation/loss": np.float32(1.5)}


def test_tensorboard_reads_the_file(tmp_path):
    loader_mod = pytest.importorskip("tensorboard.backend.event_processing.event_file_loader")
    w = S.EventWriter(str(tmp_path))
    vals = np.random.RandomState(1).normal(size=200).astype(np.float32)
    stats, counts = _histogram_of(vals)
    w.add(3, [("loss/latent_loss_1", 0.125)], [("x/bias", S.encode_histogram(stats, counts, S.bucket_limits()))])
    w.close()
    # LegacyEventFileLoader: the events as stored (EventFileLoader also migrates histograms to tensor summaries)
    loader = getattr(loader_mod, "LegacyEventFileLoader", loader_mod.EventFileLoader)
    events = list(loader(w.path).Load())
    # ... and what TensorBoard's own loader makes of them: the tags it shows, at the step written
    migrated = {v.tag: e.step for e in loader_mod.EventFileLoader(w.path).Load() for v in e.summary.value}
    assert migrated == {"loss/latent_loss_1": 3, "x/bias": 3}
    assert events[0].file_version == "brain.Event:2"
    mn, mx, num, sm, sq, lim, cnt = SO.tf_histogram(vals).encode()
    got = {}
    for e in events[1:]:
        assert e.step == 3
        for v in e.summary.value:
            got[v.tag] = v
    if got["loss/latent_loss_1"].HasField("simple_value"):
        assert got["loss/latent_loss_1"].simple_value == np.float32(0.125)
    h = got["x/bias"].histo
    assert (h.min, h.max, h.num) == (mn, mx, num)
    assert abs(h.sum - sm) <= 1e-12 * np.abs(vals).sum() and abs(h.sum_squares - sq) <= 1e-12 * sq
    assert list(h.bucket_limit) == lim and list(h.bucket) == cnt


def test_remove_event_files_leaves_everything_else(tmp_path):
    d = tmp_path / "run"
    (d / "sub").mkdir(parents=True)
    (d / "events.out.tfevents.0000000001.host").write_bytes(b"")
    (d / "sub" / "events.out.tfevents.0000000002.host").write_bytes(b"")
    (d / "notes.txt").write_text("keep")
    S.remove_event_files(str(d))
    assert sorted(os.listdir(d)) == ["notes.txt", "sub"]
    assert os.listdir(d / "sub") == ["events.out.tfevents.0000000002.host"]


def test_scalar_tags():
    """tf.summary.scalar inside loss()'s `with tf.name_scope('loss')` (lib/models.py:355): `reconstruction_loss` and
    `latent_loss` were opened as name scopes at :356 and :370, so summary_scope uniquifies them to `_1`; the rest are
    new names.  The averages sit in `loss/averages` (:407), the learning rates in `training` (:421,443-444); the edge
    loss has no summary.  fit adds `validation/loss` (:920)."""
    assert S.SCALAR_TAGS == ("loss/reconstruction_loss_1", "loss/latent_loss_1", "loss/fc_regularization_g",
                             "loss/fc_regularization_d", "loss/gan_loss_generator", "loss/gan_loss_discriminator",
                             "loss/averages/loss_g", "loss/averages/loss_d", "training/lr_g", "training/lr_d")
    assert S.VALIDATION_TAG == "validation/loss"


def _inventory_cases():
    import make_histogram_inventory as HI
    return HI.configs()


def _specs(cfg, h):
    from cape_b200.params import param_specs
    return param_specs(cfg, [l.shape[0] for l in h["L"]], [l.shape[0] for l in h["L_d"]])


@pytest.mark.parametrize("tag", ["affine_nz64", "groupnorm_nz18", "default", "plain_decoder"])
def test_histogram_inventory_is_the_references(hierarchy, tag):
    """The names the reference's own build_graph histograms (tests/golden/histogram_inventory.json, recorded by
    make_histogram_inventory.py) == summary.histogram_names(param_specs): every graph-conv weight and bias, no dense
    layer, no GroupNorm gamma / beta.  The reference histograms the discriminator once per call (real and fake) under
    the same variable name; the set is what is compared."""
    cfg = dict(_inventory_cases())[tag]
    with open(os.path.join(HERE, "golden", "histogram_inventory.json")) as f:
        ref = json.load(f)[tag]
    ours = S.histogram_names(_specs(cfg, hierarchy))
    assert len(ours) == len(set(ours))
    assert set(ours) == set(ref)
    assert not any("/dense/" in n or n.endswith("/gamma") or n.endswith("/beta") for n in ours)


@pytest.mark.skipif(not os.environ.get("CAPE_REFERENCE"), reason="needs $CAPE_REFERENCE (a reference checkout)")
@pytest.mark.parametrize("tag", ["affine_nz64", "groupnorm_nz18", "default", "plain_decoder"])
def test_reference_rerun_matches_the_inventory(hierarchy, tag):
    import make_histogram_inventory as HI
    cfg = dict(HI.configs())[tag]
    names = HI.reference_histograms(cfg, dict(hierarchy))
    with open(os.path.join(HERE, "golden", "histogram_inventory.json")) as f:
        assert names == json.load(f)[tag]
    assert set(names) == set(S.histogram_names(_specs(cfg, hierarchy)))


def test_loss_average_recurrence():
    """The host transcription: 1 - 0.9 is taken in float32 (TF's `1.0 - decay` on a float32 tensor), every operation
    rounds to float32, the shadow starts at 0 and converges to a constant loss."""
    cfg = dict(lambda_gan=0.1, lambda_recon=1.0, lambda_edge=1.0, lambda_latent=8e-4, regularization=2e-3)
    one = [([0.5, 0.25, 3.0, 0.7, 0.6, 0.8, 0, 0], 1000.0)]
    g, d = SO.loss_totals(*one[0], cfg)
    reg = np.float32(2e-3) * (np.float32(2e-3) * np.float32(500.0))
    assert g == np.float32(np.float32(np.float32(np.float32(np.float32(0.7) * np.float32(0.1)) + np.float32(0.5))
                                      + np.float32(0.25)) + np.float32(3.0) * np.float32(8e-4)) + reg
    assert d == (np.float32(0.6) + np.float32(0.8)) * np.float32(0.1)
    k = np.float32(1.0) - np.float32(0.9)
    assert k == np.float32(0.100000024)
    s = SO.loss_average(one, cfg)
    assert s[0] == np.float32(g * k) and s[1] == np.float32(d * k)
    many = SO.loss_average(one * 400, cfg)
    assert abs(many[0] - g) <= 1e-6 * g and abs(many[1] - d) <= 1e-6 * d
    assert all(isinstance(v, np.float32) for v in many)
