"""CUDA mirror of ``openwakeword.Model`` (openwakeword/model.py:32-504).

Same constructor keywords, ``predict`` / ``predict_clip`` / ``reset`` semantics, attribute names
(``models``, ``model_inputs``, ``model_outputs``, ``class_mapping``, ``prediction_buffer``,
``preprocessor``) and ``ValueError`` behaviour; the three inference sessions and the buffers between
them are replaced by one libowwb200 step per call.  Additions: ``n_streams`` independent streams on
the batch axis (``predict`` then takes ``[n_streams, samples]`` and returns arrays per label),
``predict_clips`` (array-input bulk path) and ``feature_init``.
"""
import os
import pickle
import time
from collections import defaultdict, deque
from functools import partial

import numpy as np

from . import _native
from . import weights as _weights
from .utils import AudioFeatures, re_arg, _read_wav, CHUNK, _torch
from . import registry as _registry


def _load_head_file(path):
    """-> (head dict, class mapping or None).  ``.npz`` = weights.save_head container; ``.onnx`` = a reference head
    file (torch.onnx.export of train.py's DNN family), read without the onnx package (onnx_io.py)."""
    if path.endswith(".npz"):
        return _weights.load_head(path)
    if path.endswith(".onnx"):
        from .onnx_io import head_from_onnx
        return head_from_onnx(path), None
    raise ValueError(f"unsupported model file '{path}'")


class Model:
    @re_arg({"wakeword_model_paths": "wakeword_models"})
    def __init__(self, wakeword_models=[], class_mapping_dicts=[], enable_speex_noise_suppression=False,
                 vad_threshold=0, custom_verifier_models={}, custom_verifier_threshold=0.1,
                 inference_framework="b200", **kwargs):
        if inference_framework != "b200":
            raise ValueError(f"openwakeword_b200.Model only provides inference_framework='b200' (got '{inference_framework}')")
        pretrained_paths = _registry.get_pretrained_model_paths(inference_framework)
        wakeword_models = list(wakeword_models)
        names = []
        if wakeword_models == []:
            wakeword_models = pretrained_paths
            names = list(_registry.MODELS.keys())
        else:
            for ndx, item in enumerate(wakeword_models):
                if isinstance(item, dict):                     # in-memory head: {"name":..., "head":..., "class_mapping":...}
                    names.append(item["name"])
                elif os.path.exists(item):
                    names.append(os.path.splitext(os.path.basename(item))[0])
                else:
                    match = [p for p in pretrained_paths if item.replace(" ", "_") in p.split(os.path.sep)[-1]]
                    if not match:
                        raise ValueError("Could not find pretrained model for model name '{}'".format(item))
                    wakeword_models[ndx] = match[0]
                    names.append(item)

        self.models = {}
        self.model_inputs = {}
        self.model_outputs = {}
        self.model_prediction_function = {}
        self.class_mapping = {}
        self.custom_verifier_models = {}
        self.custom_verifier_threshold = custom_verifier_threshold

        if enable_speex_noise_suppression:
            from speexdsp_ns import NoiseSuppression     # same optional dependency as the reference (model.py:200-205)
            self.speex_ns = NoiseSuppression.create(160, 16000)
        else:
            self.speex_ns = None
        self.vad_threshold = vad_threshold
        if vad_threshold > 0:
            raise ValueError("vad_threshold > 0 needs the Silero VAD ONNX model and onnxruntime, which the b200 "
                             "backend does not ship (SURVEY.md section 2 #7); run VAD outside and gate the scores")

        # feature pipeline + device context (weights are registered on its handle)
        self.preprocessor = AudioFeatures(inference_framework=inference_framework, **kwargs)
        self.n_streams = self.preprocessor.n_streams
        ctx = self.preprocessor.ctx

        self._columns = {}     # model name -> (col0, n_out)
        col = 0
        for ndx, (src, name) in enumerate(zip(wakeword_models, names)):
            if isinstance(src, dict):
                head, file_map = src["head"], src.get("class_mapping")
            else:
                if ".tflite" in src:
                    raise ValueError("The b200 inference framework is selected, but tflite models were provided!")
                if not os.path.exists(src):
                    raise ValueError(f"Model file '{src}' not found (the reference's released heads are download-only)")
                head, file_map = _load_head_file(src)
            if _weights.is_gated(head):
                # conditional verifier pair (the released hey_jarvis graph): two networks on the device, the verifier's
                # score replacing the main one's above the threshold inside the step; its own column stays hidden
                n_in, dims, ln, fin = _weights.head_desc(head["main"])
                hid = ctx.add_head(n_in, dims, ln, fin, _weights.pack_head_blob(head["main"]))
                v_in, v_dims, v_ln, v_fin = _weights.head_desc(head["verifier"])
                if v_in != n_in or dims[-1] != 1 or v_dims[-1] != 1:
                    raise ValueError(f"model '{name}': a verifier pair needs two single-output networks on the same input")
                vid = ctx.add_head(v_in, v_dims, v_ln, v_fin, _weights.pack_head_blob(head["verifier"]))
                ctx.add_gate(hid, vid, head["threshold"])
                self.model_prediction_function[name] = partial(self._gated_predict, hid, vid, n_in, head["threshold"])
                width = 2
            else:
                n_in, dims, ln, fin = _weights.head_desc(head)
                hid = ctx.add_head(n_in, dims, ln, fin, _weights.pack_head_blob(head))
                self.model_prediction_function[name] = partial(self._head_predict, hid, n_in, dims[-1])
                width = dims[-1]
            self.models[name] = hid
            self.model_inputs[name] = n_in
            self.model_outputs[name] = dims[-1]
            self._columns[name] = (col, dims[-1])
            col += width
            if class_mapping_dicts and ndx < len(class_mapping_dicts) and class_mapping_dicts[ndx].get(name, None):
                self.class_mapping[name] = class_mapping_dicts[ndx]
            elif _registry.model_class_mappings.get(name, None):
                self.class_mapping[name] = _registry.model_class_mappings[name]
            elif file_map:
                self.class_mapping[name] = file_map
            else:
                self.class_mapping[name] = {str(i): str(i) for i in range(0, dims[-1])}
            if isinstance(custom_verifier_models, dict) and custom_verifier_models.get(name, False):
                with open(custom_verifier_models[name], "rb") as fh:
                    self.custom_verifier_models[name] = pickle.load(fh)
        if len(self.custom_verifier_models.keys()) < len(custom_verifier_models.keys()):
            raise ValueError("Custom verifier models were provided, but some were not matched with a base model!"
                             " Make sure that the keys provided in the `custom_verifier_models` dictionary argument"
                             " exactly match that of the `.models` attribute of an instantiated Model object.")
        self._n_cols = col
        self._scores = np.zeros((self.n_streams, max(col, 1)), np.float32)
        self._reset_history()

    # ---- per-label history (model.py:198; vectorised over streams) ----
    def _reset_history(self):
        self._hist = {}        # label -> float32 [30, B] ring of the last predictions
        self._count = {}       # label -> int64 [B] predictions appended so far

    def _h(self, label):
        if label not in self._hist:
            self._hist[label] = np.zeros((30, self.n_streams), np.float32)
            self._count[label] = np.zeros(self.n_streams, np.int64)
        return self._hist[label], self._count[label]

    def _recent(self, label, n):
        """last n appended predictions per stream -> [<=n, B] oldest first (deque(maxlen=30) view)."""
        hist, cnt = self._h(label)
        c = int(cnt[0])                      # streams advance in lockstep
        k = min(n, c, 30)
        idx = [(c - k + i) % 30 for i in range(k)]
        return hist[idx]

    @property
    def prediction_buffer(self):
        """defaultdict(deque(maxlen=30)) of stream 0's history, like the reference attribute."""
        buf = defaultdict(partial(deque, maxlen=30))
        for label in self._hist:
            for v in self._recent(label, 30)[:, 0]:
                buf[label].append(float(v))
        return buf

    def get_parent_model_from_label(self, label):
        parent = ""
        for mdl in self.class_mapping.keys():
            if label in self.class_mapping[mdl].values():
                parent = mdl
            elif label in self.class_mapping.keys() and label == mdl:
                parent = mdl
        return parent

    def reset(self, feature_init=None):
        """model.py:226-230."""
        self._reset_history()
        self.preprocessor.reset(feature_init)

    def _head_predict(self, hid, n_in, n_out, x):
        """model_prediction_function[name]: float32 [N,n_in,96] -> [array [N,n_out]] (model.py:137-138)."""
        torch = _torch()
        x = np.ascontiguousarray(np.asarray(x, np.float32).reshape(-1, n_in, 96))
        dev = f"cuda:{self.preprocessor.device_index}"
        d = torch.from_numpy(x).to(dev)
        out = torch.empty((x.shape[0], n_out), dtype=torch.float32, device=dev)
        self.preprocessor.ctx.head_predict(hid, d, x.shape[0], out, torch.cuda.current_stream(d.device).cuda_stream)
        return [out.cpu().numpy()]

    def _gated_predict(self, hid, vid, n_in, thr, x):
        p1 = self._head_predict(hid, n_in, 1, x)[0]
        p2 = self._head_predict(vid, n_in, 1, x)[0]
        return [np.where(p1 > np.float32(thr), p2, p1).astype(np.float32)]

    def _suppress_noise_with_speex(self, x, frame_size=160):
        cleaned = [self.speex_ns.process(x[i:i + frame_size].tobytes()) for i in range(0, x.shape[0], frame_size)]
        return np.frombuffer(b"".join(cleaned), np.int16)

    def predict(self, x, patience={}, threshold={}, debounce_time=0.0, timing=False):
        """One streaming step (model.py:232-386).  x: ndarray [samples] (n_streams == 1) or
        [n_streams, samples].  Returns {label: float} for a single stream, {label: float32[B]} otherwise."""
        if not isinstance(x, np.ndarray):
            raise ValueError(f"The input audio data (x) must by a Numpy array, instead received an object of type {type(x)}.")
        single = self.n_streams == 1
        if timing:
            timing_dict = {"models": {}}
            t0 = time.time()
        if self.speex_ns:
            if not single:
                raise ValueError("Speex noise suppression is single-stream")
            x = self._suppress_noise_with_speex(x)
        n_prepared, n_chunks = self.preprocessor._streaming_features(x, self._scores)
        if timing:
            timing_dict["models"]["preprocessor"] = time.time() - t0

        B = self.n_streams
        predictions = {}
        for mdl in self.models.keys():
            if timing:
                t1 = time.time()
            col0, n_out = self._columns[mdl]
            if n_prepared >= CHUNK:
                pred = self._scores[:, col0:col0 + n_out]            # max over chunk windows done on device
            elif n_out == 1:
                hist, cnt = self._h(mdl)
                pred = (hist[(int(cnt[0]) - 1) % 30] if cnt[0] > 0 else np.zeros(B, np.float32))[:, None]
            else:
                n_classes = max(int(i) for i in self.class_mapping[mdl].keys())
                pred = np.zeros((B, n_classes + 1), np.float32)
            if n_out == 1:
                predictions[mdl] = pred[:, 0].copy()
            else:
                for int_label, cls in self.class_mapping[mdl].items():
                    predictions[cls] = pred[:, int(int_label)].copy()

            if self.custom_verifier_models != {}:
                for cls in list(predictions.keys()):
                    parent = self.get_parent_model_from_label(cls)
                    if self.custom_verifier_models.get(parent, False):
                        for b in np.nonzero(predictions[cls] >= self.custom_verifier_threshold)[0]:
                            feats = self.preprocessor.get_features(self.model_inputs[mdl], stream=int(b))
                            predictions[cls][b] = self.custom_verifier_models[parent].predict_proba(feats)[0][-1]

            for cls in predictions.keys():                            # model.py:330-333
                _, cnt = self._h(cls)
                predictions[cls] = np.where(cnt < 5, np.float32(0.0), predictions[cls])
            if timing:
                timing_dict["models"][mdl] = time.time() - t1

        if patience != {} or debounce_time > 0:
            if threshold == {}:
                raise ValueError("Error! When using the `patience` argument, threshold "
                                 "values must be provided via the `threshold` argument!")
            if patience != {} and debounce_time > 0:
                raise ValueError("Error! The `patience` and `debounce_time` arguments cannot be used together!")
            for lab in predictions.keys():
                parent = self.get_parent_model_from_label(lab)
                nz = predictions[lab] != 0.0
                if parent in patience.keys():
                    sc = self._recent(lab, patience[parent])
                    fail = (sc >= threshold[parent]).sum(axis=0) < patience[parent]
                    predictions[lab] = np.where(nz & fail, np.float32(0.0), predictions[lab])
                elif debounce_time > 0 and parent in threshold.keys():
                    n_frames = int(np.ceil(debounce_time / (n_prepared / 16000)))
                    rec = self._recent(lab, n_frames)
                    hit = (rec >= threshold[parent]).sum(axis=0) > 0
                    predictions[lab] = np.where(nz & (predictions[lab] >= threshold[parent]) & hit,
                                                np.float32(0.0), predictions[lab])

        for lab in predictions.keys():
            hist, cnt = self._h(lab)
            hist[int(cnt[0]) % 30] = predictions[lab]
            cnt += 1

        out = {k: (float(v[0]) if single else v) for k, v in predictions.items()}
        if timing:
            return out, timing_dict
        return out

    def predict_clip(self, clip, padding=1, chunk_size=1280, **kwargs):
        """model.py:388-426: path or int16 array -> list of per-step dicts (no reset, like the reference)."""
        if isinstance(clip, str):
            data = _read_wav(clip)
        elif isinstance(clip, np.ndarray):
            data = clip
        else:
            raise ValueError("clip must be a WAV path or a numpy array")
        if self.n_streams != 1:
            raise ValueError("predict_clip is single-stream; use predict_clips for batches")
        if padding:
            z = np.zeros(16000 * padding).astype(np.int16)
            data = np.concatenate((z, data, z))
        return [self.predict(data[i:i + chunk_size], **kwargs) for i in range(0, data.shape[0] - chunk_size, chunk_size)]

    def _get_positive_prediction_frames(self, file, threshold=0.5, return_type="features", **kwargs):
        """model.py:428-478: run the WAV through ``predict`` in 1280-sample steps and collect, per label, what produced
        a score >= ``threshold``: the head's input features ``[n_in, 96]`` at that step (``return_type="features"``) or
        the 4 s of audio around it (``"audio"``: 3 s before, 1 s after; steps without a full 4 s are dropped).
        Returns {label: stacked array}; labels without a hit are absent."""
        if return_type not in ("features", "audio"):
            raise ValueError("return_type must be 'features' or 'audio'")
        if self.n_streams != 1:
            raise ValueError("_get_positive_prediction_frames is single-stream")
        data = _read_wav(file)
        hits = defaultdict(list)
        for i in range(0, data.shape[0] - CHUNK, CHUNK):
            for lbl, score in self.predict(data[i:i + CHUNK], **kwargs).items():
                if score < threshold:
                    continue
                if return_type == "features":
                    parent = self.get_parent_model_from_label(lbl)
                    hits[lbl].append(self.preprocessor.get_features(self.model_inputs[parent]))
                else:
                    context = data[max(0, i - 16000 * 3):i + 16000]
                    if len(context) == 16000 * 4:
                        hits[lbl].append(context)
        return {lbl: np.vstack(v) for lbl, v in hits.items() if v}

    def predict_clips(self, clips, padding=1, feature_init=None):
        """Array-input bulk path (extension; SURVEY.md F9): int16 [N,S] equal-length clips, each from a
        fresh state, 1280-sample steps.  Returns a list (per clip) of lists (per step) of {label: float},
        i.e. what predict_clip would return for each clip after reset(feature_init)."""
        scores, labels = self.predict_clips_array(clips, padding, feature_init)
        return [[{lab: float(scores[c, s, j]) for j, lab in enumerate(labels)} for s in range(scores.shape[1])]
                for c in range(scores.shape[0])]

    def labels(self):
        """Output labels in score-column order (binary heads: model name; multi-class: mapped labels)."""
        labs = []
        for mdl in self.models:
            if self.model_outputs[mdl] == 1:
                labs.append(mdl)
            else:
                labs += list(self.class_mapping[mdl].values())
        return labs

    def predict_clips_array(self, clips, padding=1, feature_init=None):
        """-> (float32 [N, steps, n_labels], labels) with the first-5-steps zeroing of model.py:330-333 applied."""
        torch = _torch()
        if isinstance(clips, torch.Tensor):            # CPU (ideally pinned) or CUDA int16 tensor: no host copy
            if clips.dtype != torch.int16:
                clips = clips.to(torch.int16)
            clips = clips.contiguous()
        else:
            clips = np.ascontiguousarray(np.asarray(clips))
            if clips.dtype != np.int16:
                clips = clips.astype(np.int16)
        N, S = clips.shape
        L = S + 2 * 16000 * padding
        steps = len(range(0, L - CHUNK, CHUNK))
        fi = feature_init if feature_init is not None else self.preprocessor._feature_init
        if fi is None:
            fi = self.preprocessor._get_embeddings(np.random.randint(-1000, 1000, 16000 * 4).astype(np.int16))
        dev = f"cuda:{self.preprocessor.device_index}"
        d = clips.to(dev, non_blocking=True) if isinstance(clips, torch.Tensor) else torch.from_numpy(clips).to(dev)
        raw = torch.zeros((N, steps, max(self._n_cols, 1)), dtype=torch.float32, device=dev)
        self.preprocessor.ctx.predict_clips(d, N, S, 16000 * padding, fi, raw, torch.cuda.current_stream(d.device).cuda_stream)
        raw = raw.cpu().numpy()
        cols, labels = [], []
        for mdl in self.models:
            col0, n_out = self._columns[mdl]
            if n_out == 1:
                cols.append(col0); labels.append(mdl)
            else:
                for k, lab in self.class_mapping[mdl].items():
                    cols.append(col0 + int(k)); labels.append(lab)
        out = raw[:, :, cols]
        out[:, :5, :] = 0.0
        return out, labels
