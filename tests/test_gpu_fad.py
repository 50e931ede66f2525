"""GPU, end to end: vampnet_b200.fad with seeded random VGGish weights against the float64 oracle's goldens
(tests/golden/fad_*.npz, oracle/gen_fad_golden.py), batching, host syncs, refusals and the eval CLI's frechet column."""
import csv

import numpy as np
import pytest
import torch

from oracle import fad_oracle as fo
from vampnet_b200 import _lib, fad
from vampnet_b200.audio import AudioSignal

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLDEN = "tests/golden/fad_tones.npz"
# |kernel - float64| / max |float64| of the embeddings: nine layers of the per-layer bounds of test_gpu_fad_ops.py,
# dominated by the first fully connected layer's K 2^-24 rss at K = 12288 (measured on an H100: DESIGN.md §14)
EMB_TOL = 1e-3
SCORE_TOL = 1e-3  # relative, on the distance


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


@pytest.fixture(scope="module")
def model(golden):
    return fad.FrechetAudioDistance(fo.random_state_dict(int(golden["seed"])), device=DEV)


def _signals(golden, side):
    x = golden[f"{side}_signal"].astype(np.float32)
    cuts = np.cumsum(golden[f"{side}_lengths"])[:-1]
    return [torch.from_numpy(s.copy()).to(DEV) for s in np.split(x, cuts)]


def test_score_matches_oracle(golden, model):
    moms = []
    for side in ("background", "eval"):
        e = model.embeddings(_signals(golden, side))
        want = golden[f"{side}_embeddings"]
        assert e.shape == want.shape
        err = np.abs(e.double().cpu().numpy() - want).max() / np.abs(want).max()
        print(f"{side}: embeddings within {err:.2e} of float64")
        assert err <= EMB_TOL
        moms.append(fad.moments(e))
    got = model.score_moments(*moms)
    rel = abs(got - float(golden["score"])) / float(golden["score"])
    print(f"score {got!r} oracle {float(golden['score'])!r} rel {rel:.2e}")
    assert rel <= SCORE_TOL


def test_batch_embeds_bit_identically_to_each_example_alone(golden, model):
    ex = torch.cat([model.model.examples(s) for s in _signals(golden, "eval")])
    batch = model.model.embed(ex)
    for i in range(ex.shape[0]):
        assert torch.equal(model.model.embed(ex[i:i + 1].clone()), batch[i:i + 1])
    old = fad.MAX_BATCH
    try:
        fad.MAX_BATCH = 4  # several launches, a partial last one
        assert torch.equal(model.model.embed(ex), batch)
    finally:
        fad.MAX_BATCH = old


def test_no_host_sync(golden, model):
    sigs = _signals(golden, "background")
    model.embeddings(sigs)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        mu, sigma = fad.moments(model.embeddings(sigs))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert mu.shape == (128,) and sigma.shape == (128, 128)


def test_refusals(tmp_path):
    sd = fo.random_state_dict(2, pproc=True)
    path = tmp_path / "vggish.pth"
    torch.save(sd, path)
    v = fad.VGGish.load(path, device=DEV)  # pproc.* is ignored
    assert v.embed(torch.zeros(0, 96, 64, device=DEV)).shape == (0, 128)
    bad = dict(sd)
    bad["features.0.weight"] = torch.zeros(64, 1, 3, 4)
    torch.save(bad, tmp_path / "bad.pth")
    with pytest.raises(ValueError):
        fad.VGGish.load(tmp_path / "bad.pth", device=DEV)
    with pytest.raises(ValueError):
        fad.FrechetAudioDistance(path, use_pca=True)
    with pytest.raises(ValueError):
        fad.FrechetAudioDistance(path, use_activation=True)
    one = fad.FrechetAudioDistance(v).embeddings([torch.zeros(15600, device=DEV)])
    with pytest.raises(ValueError):
        fad.moments(one)
    import ctypes as C
    L = _lib.lib()
    w = _lib.VggishWeights()
    assert L.vnb_vggish_create(w, None) != 0
    hd = C.c_void_p()
    assert L.vnb_vggish_create(C.byref(w), C.byref(hd)) != 0 and b"NULL" in L.vnb_last_error()
    n = C.c_uint64()
    assert L.vnb_vggish_workspace_bytes(0, C.byref(n)) != 0
    assert L.vnb_vggish_embed(None, None, 1, None, 0, None, _lib.stream_ptr()) != 0


def test_eval_cli_frechet(tmp_path):
    from vampnet_b200 import eval as ev
    sd = fo.random_state_dict(3, pproc=True)
    ckpt = tmp_path / "vggish.pth"
    torch.save(sd, ckpt)
    exp = tmp_path / "exp"
    sr = 16000
    for d in ("baseline", "plain", "inpaint_0.5"):
        (exp / d).mkdir(parents=True)
    for i in range(3):
        x = fo.test_signal(2 * sr, 30 + i)
        y = fo.test_signal(2 * sr, 40 + i)
        AudioSignal(x[None, None], sr).write(exp / "baseline" / f"{i}.wav")
        AudioSignal((0.5 * x + 0.5 * y)[None, None], sr).write(exp / "plain" / f"{i}.wav")
        y44 = fo.test_signal(2 * 44100, 40 + i, sr=44100)  # resampled to 16 kHz by both metrics
        AudioSignal(y44[None, None], 44100).write(exp / "inpaint_0.5" / f"{i}.wav")
    ev.main(["--exp_dir", str(exp), "--vggish_ckpt", str(ckpt)])
    with open(exp / "metrics-all.csv") as f:
        rows = list(csv.reader(f))
    assert rows[0] == ["mel", "frechet", "condition", "file"]
    f = fad.FrechetAudioDistance(str(ckpt))
    for cond in ("inpaint_0.5", "plain"):
        vals = {r[1] for r in rows[1:] if r[2] == cond}
        assert len(vals) == 1 and sum(r[2] == cond for r in rows[1:]) == 3
        assert float(vals.pop()) == f.score(exp / "baseline", exp / cond)
    with open(exp / "stats-frechet.csv") as fh:
        stats = list(csv.reader(fh))
    assert stats[0] == ["condition", "mean", "count", "std"] and [r[0] for r in stats[1:]] == ["inpaint_0.5", "plain"]
    for r in stats[1:]:  # as stats-mel.csv: np.mean and np.std(ddof=1) of the condition's rows
        v = np.array([float(x[1]) for x in rows[1:] if x[2] == r[0]])
        assert float(r[1]) == v.mean() and r[2] == "3" and float(r[3]) == np.std(v, ddof=1)
    assert (exp / "stats-mel.csv").exists()
