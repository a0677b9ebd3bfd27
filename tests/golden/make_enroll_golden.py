"""Generate tests/golden/enroll_alexa.npz with the UNMODIFIED reference ``train_custom_verifier``.

    OWW_REFERENCE=/path/to/openWakeWord python tests/golden/make_enroll_golden.py

Same set-up as make_golden.py: the reference's own ``openwakeword`` package, ``oracle.ref_stub_ort`` standing in for
onnxruntime, synthetic seeded weights.  The parent is alexa_v0.1 with its output bias shifted so that its scores on the
positive clip straddle 0.5: ``bias_shift`` (minus the logit of the median nonzero score of a plain pass) is added to
its output bias, then its output layer is scaled by ``spread`` so that few scores lie near 0.5.  Positives: the
reference's alexa_test.wav and hey_jane.wav; negatives: hey_mycroft_test.wav.  Around the reference call the maker only
records - it wraps, without changing, ``np.random.randint`` (the initial feature ring and the offsets it draws, which
start the positive passes), ``get_reference_clip_features`` (negative passes, and the windows each call returns) and
``Model.predict`` (every step's score).  Windows per pass are the steps whose score meets the pass's threshold, checked
against the windows the reference returned.  Of seeds 0, 1, ... it keeps the first where no positive-pass score
lies within 2e-3 of 0.5.  Stored: the seed, the offsets, the windows captured per pass, the pickled pipeline's mean_,
var_, coef_ and intercept_, its predict_proba on a fixed probe set (windows of the three clips plus noise), the nearest
distance of a positive-pass score to 0.5, and the clips' PCM.
"""
import os
import pickle
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import make_golden as G                             # noqa: E402
from openwakeword_b200 import weights as W          # noqa: E402
from oracle import ref_stub_ort                     # noqa: E402

PARENT = "alexa_v0.1"
SPREAD = 16.0


def main():
    emb = W.synthetic_embedding(G.EMB_SEED)
    head = W.synthetic_head(**G.HEAD_SPECS[PARENT])
    ref_root = os.environ["OWW_REFERENCE"]
    sys.path.insert(0, ref_root)
    wavs = {n: G.read_wav(os.path.join(ref_root, "tests", "data", f"{n}.wav"))
            for n in ("alexa_test", "hey_jane", "hey_mycroft_test")}
    pos, neg = [wavs["alexa_test"], wavs["hey_jane"]], [wavs["hey_mycroft_test"]]
    tmp = tempfile.mkdtemp()
    paths = {k: os.path.join(tmp, k + ".onnx") for k in (PARENT, "melspectrogram", "embedding_model")}
    for p in paths.values():
        open(p, "w").close()
    kw = dict(inference_framework="onnx", melspec_model_path=paths["melspectrogram"],
              embedding_model_path=paths["embedding_model"])

    ref_stub_ort.install(emb, {PARENT: head})
    import openwakeword.custom_verifier_model as cvm                               # the reference, unmodified
    from openwakeword.model import Model

    # bias shift: centre the positive scores of one plain pass on 0.5
    np.random.seed(0)
    m = Model(wakeword_models=[paths[PARENT]], **kw)
    s = np.array([m.predict(pos[0][i:i + 1280])[PARENT] for i in range(0, len(pos[0]) - 1280, 1280)], np.float64)
    med = float(np.median(s[s > 0]))
    shift = -float(np.log(med / (1 - med)))
    last = head["layers"][-1]                      # and spread the logits, so few scores lie near 0.5
    last["b"] = ((last["b"] + np.float32(shift)) * np.float32(SPREAD)).astype(np.float32)
    last["W"] = (last["W"] * np.float32(SPREAD)).astype(np.float32)
    ref_stub_ort.install(emb, {PARENT: head})

    rand, real_grc, real_predict = np.random.randint, cvm.get_reference_clip_features, Model.predict
    originals = (rand, real_grc, real_predict)
    for seed in range(50):
        log = {"offsets": [], "ring": 0, "passes": [], "thr": [], "captured": 0}

        def randint(*a, **k):
            v = rand(*a, **k)
            if a[:2] == (0, 1280):                  # a positive pass starts
                log["offsets"].append(int(v))
                log["passes"].append([])
                log["thr"].append(0.5)
            elif a[:2] == (-1000, 1000):
                log["ring"] += 1
            return v

        def grc(clip, oww, name, threshold=0.5, N=3, **k):
            if N == 1:                              # a negative pass starts (no offset draw)
                log["passes"].append([])
                log["thr"].append(threshold)
            out = real_grc(clip, oww, name, threshold=threshold, N=N, **k)
            log["captured"] += len(out)
            return out

        def predict(self, x, *a, **k):
            r = real_predict(self, x, *a, **k)
            log["passes"][-1].append(r[PARENT])
            return r

        patched = (randint, grc, predict)
        np.random.randint, cvm.get_reference_clip_features, Model.predict = patched
        try:
            np.random.seed(seed)
            out = os.path.join(tmp, "v.pkl")
            cvm.train_custom_verifier(pos, neg, out, paths[PARENT], **kw)
        finally:
            np.random.randint, cvm.get_reference_clip_features, Model.predict = originals
        # the comparison get_reference_clip_features makes (custom_verifier_model.py:78), per pass
        counts = [int(sum(v >= t for v in p)) for p, t in zip(log["passes"], log["thr"])]
        assert sum(counts) == log["captured"], (counts, log["captured"])
        log["counts"] = counts
        log["scores"] = [v for p, t in zip(log["passes"], log["thr"]) if t == 0.5 for v in p]
        nearest = float(np.abs(np.asarray(log["scores"], np.float64) - 0.5).min())
        print(f"seed {seed}: nearest positive-pass score to 0.5 = {nearest:.2e}, counts {log['counts']}")
        if nearest >= 2e-3:
            break
    assert log["ring"] == 1 and len(log["offsets"]) == 5 * len(pos)
    with open(out, "rb") as f:
        pipe = pickle.load(f)
    sc, lr = pipe.steps[1][1], pipe.steps[2][1]
    rng = np.random.default_rng(1)
    probe_pcm = np.concatenate(pos + neg)
    np.random.seed(1234)
    m = Model(wakeword_models=[paths[PARENT]], **kw)
    probe = []
    for i in range(0, len(probe_pcm) - 1280, 1280):
        m.predict(probe_pcm[i:i + 1280])
        probe.append(m.preprocessor.get_features(16))
    probe = np.vstack(probe).astype(np.float32)
    probe = np.concatenate([probe, probe[rng.choice(len(probe), 64)] + rng.normal(0, 0.2, (64, 16, 96)).astype(np.float32)])
    np.savez_compressed(os.path.join(HERE, "enroll_alexa.npz"),
                        seed=np.int64(seed), bias_shift=np.float64(shift), spread=np.float64(SPREAD), offsets=np.array(log["offsets"], np.int64),
                        counts=np.array(log["counts"], np.int64), nearest=np.float64(nearest),
                        mean=sc.mean_, var=sc.var_, coef=lr.coef_[0], intercept=np.float64(lr.intercept_[0]),
                        probe=probe, probe_p=pipe.predict_proba(probe)[:, 1],
                        pos0=pos[0], pos1=pos[1], neg0=neg[0], emb_seed=np.int64(G.EMB_SEED))
    print("wrote enroll_alexa.npz: seed", seed, "windows", sum(log["counts"]), "probe", probe.shape)


if __name__ == "__main__":
    main()
