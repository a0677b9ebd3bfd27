"""Generate the custom-verifier fixtures tests/golden/verifier_*.{pkl,npz} with the UNMODIFIED reference plumbing.

    OWW_REFERENCE=/path/to/openWakeWord python tests/golden/make_verifier_golden.py

Same set-up as make_golden.py (the reference's own ``openwakeword`` package, ``oracle.ref_stub_ort`` standing in for
onnxruntime, synthetic seeded weights).  For a binary parent (alexa_v0.1) and a multi-class parent (the timer-like
7-output head; the reference checks verifier keys inside its model loop, so the verified model comes first) it
  1. collects the parent's input window after every step of the reference's ``predict`` (what
     ``get_reference_clip_features`` gathers at threshold 0),
     20 positives from one clip and 40 negatives from the other two (each behind 1 s of silence);
  2. trains a verifier with the reference's ``train_verifier_model`` and pickles it (verifier_<parent>.pkl), so the
     pickle names ``openwakeword.custom_verifier_model.flatten_features`` exactly as a user's file does;
  3. runs ``Model(custom_verifier_models=..., custom_verifier_threshold=thr).predict_clip`` at chunk 1280 and 2560.
The threshold is the middle of the widest gap in the middle third of the parent's nonzero unverified scores at chunk
1280, so some steps are verified and some are not, and no score lies close to it; ``n_verified`` counts the (step, label) scores of the unverified run that reach it.
Only these fixtures are written; the others stay byte-identical.
"""
import os
import pickle
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as G                             # noqa: E402
from openwakeword_b200 import weights as W          # noqa: E402
from oracle import ref_stub_ort                     # noqa: E402

CASES = {   # tag -> (loaded models, verified parent, positive clip (the other two are the negatives), seed)
    "alexa": (["alexa_v0.1"], "alexa_v0.1", "alexa_test", 21),
    "timer": (["timer_v0.1"], "timer_v0.1", "hey_mycroft_test", 22),
}


def main():
    emb = W.synthetic_embedding(G.EMB_SEED)
    heads = {k: W.synthetic_head(**v) for k, v in G.HEAD_SPECS.items()}
    ref_stub_ort.install(emb, heads)
    ref_root = os.environ["OWW_REFERENCE"]
    sys.path.insert(0, ref_root)
    from openwakeword.model import Model                                            # the reference, unmodified
    from openwakeword.custom_verifier_model import train_verifier_model

    def windows(m, parent, pcm):
        # get_reference_clip_features(pcm, m, parent, threshold=0.0, N=1) without its score lookup, which needs a
        # binary parent: the parent's input window after every 1280-sample predict step
        out = []
        for i in range(0, pcm.shape[0] - 1280, 1280):
            m.predict(pcm[i:i + 1280])
            out.append(m.preprocessor.get_features(m.model_inputs[parent]))
        return np.vstack(out)

    tmp = tempfile.mkdtemp()
    paths = {}
    for k in list(heads) + ["melspectrogram", "embedding_model"]:
        paths[k] = os.path.join(tmp, k + ".onnx")
        open(paths[k], "w").close()

    def make_model(names, seed, **kw):
        np.random.seed(seed)
        m = Model(wakeword_models=[paths[n] for n in names], inference_framework="onnx",
                  melspec_model_path=paths["melspectrogram"], embedding_model_path=paths["embedding_model"], **kw)
        if "timer_v0.1" in names:
            m.class_mapping["timer_v0.1"] = dict(G.TIMER_MAP)
        return m, m.preprocessor.feature_buffer.astype(np.float32).copy()

    wavs = {n: G.read_wav(os.path.join(ref_root, "tests", "data", f"{n}.wav"))
            for n in ("alexa_test", "hey_mycroft_test", "hey_jane")}
    cases = {}
    for tag, (names, parent, pos_clip, seed) in CASES.items():
        z = np.zeros(16000, np.int16)
        m, _ = make_model(names, seed)
        pos = windows(m, parent, np.concatenate((z, wavs[pos_clip], z)))
        m.reset()
        neg = windows(m, parent, np.concatenate([z] + [wavs[n] for n in wavs if n != pos_clip]))
        rng = np.random.default_rng(seed)
        pos = pos[rng.choice(len(pos), 20, replace=False)]
        neg = neg[rng.choice(len(neg), 40, replace=False)]
        pipe = train_verifier_model(np.vstack((pos, neg)), np.array([1] * len(pos) + [0] * len(neg)))
        pkl = os.path.join(HERE, f"verifier_{tag}.pkl")
        with open(pkl, "wb") as f:
            pickle.dump(pipe, f)

        m, _ = make_model(names, seed)
        plain = m.predict_clip(wavs[pos_clip], chunk_size=1280)
        parent_labels = [parent] if parent != "timer_v0.1" else list(G.TIMER_MAP.values())
        vals = np.array([[r[lab] for lab in parent_labels] for r in plain], np.float32)
        v = np.sort(vals[vals > 0]).astype(np.float64)  # the middle of the widest gap in the middle third of the scores
        k = len(v) // 3 + int(np.argmax(np.diff(v[len(v) // 3:2 * len(v) // 3 + 1])))
        thr = float((v[k] + v[k + 1]) / 2)
        print(tag, "threshold", thr, "nearest score", float(np.abs(v - thr).min()))
        for chunk in (1280, 2560):
            m, fi = make_model(names, seed)
            plain = m.predict_clip(wavs[pos_clip], chunk_size=chunk)
            n_verified = int(sum(np.float32(r[lab]) >= np.float32(thr) for r in plain for lab in parent_labels))
            m, fi = make_model(names, seed, custom_verifier_models={parent: pkl}, custom_verifier_threshold=thr)
            res = m.predict_clip(wavs[pos_clip], chunk_size=chunk)
            labels = list(res[0].keys())
            c = dict(kind="verifier_clip", names=names, parent=parent, verifier=os.path.basename(pkl), pcm=wavs[pos_clip],
                     feature_init=fi, chunk=chunk, padding=1, labels=labels, threshold=np.float64(thr),
                     n_verified=np.int64(n_verified), kw={},
                     scores=np.array([[r[lab] for lab in labels] for r in res], dtype=np.float32),
                     unverified=np.array([[r[lab] for lab in labels] for r in plain], dtype=np.float32))
            cases[f"verifier_{tag}_c{chunk}"] = c
            print(f"verifier_{tag}_c{chunk}", c["scores"].shape, "threshold", thr, "verified", n_verified)
    G.write_cases(cases, HERE)


if __name__ == "__main__":
    main()
