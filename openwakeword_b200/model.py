"""CUDA mirror of ``openwakeword.Model`` (openwakeword/model.py:32-504).

Same constructor keywords, ``predict`` / ``predict_clip`` / ``reset`` semantics, attribute names
(``models``, ``model_inputs``, ``model_outputs``, ``class_mapping``, ``prediction_buffer``,
``preprocessor``) and ``ValueError`` behaviour; the three inference sessions and the buffers between
them are replaced by one libowwb200 step per call.  Additions: ``n_streams`` independent streams on
the batch axis (``predict`` then takes ``[n_streams, samples]`` and returns arrays per label),
``predict_clips`` / ``predict_clips_ragged`` (bulk path over clips of any lengths) and ``feature_init``.  ``sr`` (passed
to ``AudioFeatures``) other than 16000 makes ``predict*`` and ``detect*`` take each stream's audio at its own rate,
resampled on the device (``set_sample_rates`` changes it); the clip and bulk paths then refuse clips without an ``sr``
of their own.  Those paths take ``sr=`` (one rate or one per clip) on any Model, and WAV paths their header's rate:
the clips are resampled to 16 kHz on the device with their padding (``AudioFeatures.resample_clips``) and run as
16 kHz clips, which is what a fresh stream at that rate makes of the padded clip.
"""
import os
import time
import warnings
from collections import defaultdict, deque
from functools import partial

import numpy as np

from . import _native
from . import weights as _weights
from .utils import AudioFeatures, re_arg, _read_wav, _read_wav_rate, CHUNK, _torch
from . import registry as _registry
from .custom_verifier_model import load_verifier, linear_verifier_params


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
                 inference_framework="b200", stream_models={}, stream_model_capacity=256, stream_verifiers={}, **kwargs):
        """stream_models: {name: {stream id or None (every stream): model}} - a model per stream under one label
        (``set_stream_model``); stream_model_capacity: distinct models each such name can hold at once;
        stream_verifiers: {name of stream_models: {stream id or None: verifier}} (``set_stream_verifier``)."""
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
        self._host_verifiers = {}      # parent -> verifier run per stream on the host (not device-runnable)
        self._vbanks = {}              # parent -> {"bank", "slots" int32[B], "objs"}: verifiers on the device (verifier.cu)
        self._svbanks = {}             # stream-model name -> the same, for a verifier bank of its head bank
        self.stream_verifiers = {}     # stream-model name -> verifier, or {stream id: verifier} (set_stream_verifier)
        self.custom_verifier_threshold = custom_verifier_threshold
        self._head_ids = {}            # parent -> head id a verifier bank attaches to (a gated pair: its main head)
        device_verifiers = {}          # parent -> {stream id or None (all): verifier}

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
        self._check_speex_rates()
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
                self._head_ids[name] = hid
                self.model_prediction_function[name] = partial(self._gated_predict, hid, vid, n_in, head["threshold"])
                width = 2
            else:
                n_in, dims, ln, fin = _weights.head_desc(head)
                hid = ctx.add_head(n_in, dims, ln, fin, _weights.pack_head_blob(head))
                self._head_ids[name] = hid
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
                spec = custom_verifier_models[name]
                if isinstance(spec, dict):              # {stream id: path or pipeline}: device-runnable only
                    device_verifiers[name] = dict(spec)
                    self.custom_verifier_models[name] = spec
                else:                                   # the reference form: one verifier for every stream
                    v = load_verifier(spec)
                    self.custom_verifier_models[name] = v
                    if self._device_params(name, v) is not None:
                        device_verifiers[name] = {None: v}
                    else:
                        self._host_verifiers[name] = v
        self._sbanks = {}              # name -> per-stream head bank state (set_stream_model)
        for name, per_stream in stream_models.items():
            if name in self.models:
                raise ValueError(f"stream model name '{name}' is also a wakeword_models name")
            if name in custom_verifier_models:
                raise ValueError(f"custom verifier models apply to wakeword_models, not to the stream models '{name}'")
            models = [m for m in per_stream.values() if m is not None]
            if not models:
                raise ValueError(f"stream models '{name}': no model given, so the shape is unknown")
            first = per_stream[None] if per_stream.get(None) is not None else models[0]
            head, file_map = self._read_stream_model(first)
            n_in, dims, ln, fin = _weights.head_desc(head)
            bank = ctx.add_head_bank(n_in, dims, ln, fin, stream_model_capacity)
            self._sbanks[name] = {"bank": bank, "shape": (n_in, list(dims), ln, fin), "capacity": stream_model_capacity,
                                  "slots": None, "keys": None}
            self.models[name] = bank
            self.model_inputs[name] = n_in
            self.model_outputs[name] = dims[-1]
            self.model_prediction_function[name] = partial(self._bank_predict, name, n_in, dims[-1])
            self._columns[name] = (col, dims[-1])
            col += dims[-1]
            if dims[-1] == 1:
                self.class_mapping[name] = {"0": name}
            else:
                self.class_mapping[name] = file_map or {str(i): str(i) for i in range(0, dims[-1])}
        if len(self.custom_verifier_models.keys()) < len(custom_verifier_models.keys()):
            raise ValueError("Custom verifier models were provided, but some were not matched with a base model!"
                             " Make sure that the keys provided in the `custom_verifier_models` dictionary argument"
                             " exactly match that of the `.models` attribute of an instantiated Model object.")
        self._n_cols = col
        self._scores = np.zeros((self.n_streams, max(col, 1)), np.float32)
        self._reset_history()
        self._stream_det = {}          # stream id -> (threshold, patience, debounce_time) of set_stream_detection
        self._stream_det_pushed = None  # the detect call settings the device's stream settings were resolved under
        self._stream_det_on_device = False
        for name, per_stream in device_verifiers.items():
            for b, v in per_stream.items():
                self.set_custom_verifier(name, v, None if b is None else [b])
        for name, per_stream in stream_models.items():
            if None in per_stream:
                self.set_stream_model(name, per_stream[None])
            for b, m in per_stream.items():
                if b is not None:
                    self.set_stream_model(name, m, [b])
        for name, per_stream in stream_verifiers.items():
            if name not in self._sbanks:
                raise ValueError(f"stream verifiers apply to stream models; '{name}' is not one")
            if None in per_stream:
                self.set_stream_verifier(name, per_stream[None])
            for b, v in per_stream.items():
                if b is not None:
                    self.set_stream_verifier(name, v, [b])

    # ---- a model per stream (include/owwb200.h, oww_add_head_bank) ----
    @staticmethod
    def _read_stream_model(model):
        """(head dict, class mapping or None) of an .onnx / .npz path or an in-memory head dict."""
        if isinstance(model, dict):
            return model, None
        if isinstance(model, (str, os.PathLike)):
            path = os.fspath(model)
            if not os.path.exists(path):
                raise ValueError(f"Model file '{path}' not found")
            return _load_head_file(path)
        raise ValueError(f"a stream model is an .onnx / .npz path or a head dict, got {type(model)}")

    def set_stream_model(self, name, model, streams=None):
        """Run `model` (an .onnx / .npz path or a head dict of the shape of `name`'s first model; None removes it) on
        `streams` (stream ids; None = every stream) under label `name` from the next call on.  The same path or object
        on many streams shares one slot of the bank; a slot no stream uses is free again.  A stream without a model
        reads 0.0.  The streams keep their label history (``reset_streams`` starts a new client afresh)."""
        st = self._sbanks.get(name)
        if st is None:
            raise ValueError(f"no stream models named '{name}'")
        B = self.n_streams
        ids = np.arange(B) if streams is None else np.unique(np.asarray(streams, np.int64).ravel())
        if ids.size == 0:
            return
        if ids.min() < 0 or ids.max() >= B:
            raise ValueError(f"stream ids must lie in [0, {B})")
        ctx = self.preprocessor.ctx
        if st["slots"] is None:
            self.preprocessor._ensure_streams()
            st["slots"], st["keys"] = np.full(B, -1, np.int32), [None] * B
        slots, keys = st["slots"], st["keys"]
        slot = -1
        key = None
        if model is not None:
            key = os.fspath(model) if isinstance(model, (str, os.PathLike)) else model
            others = np.ones(B, bool)
            others[ids] = False
            live = {int(slots[b]): keys[b] for b in np.nonzero(others & (slots >= 0))[0]}
            same = [k for k, v in live.items() if v is key or (isinstance(key, str) and v == key)]
            if same:
                slot = same[0]
            else:
                head, _ = self._read_stream_model(model)
                n_in, dims, ln, fin = _weights.head_desc(head)
                if (n_in, list(dims), ln, fin) != st["shape"]:
                    raise ValueError(f"stream models '{name}' have the shape {st['shape']}, got {(n_in, list(dims), ln, fin)}")
                free = [k for k in range(st["capacity"]) if k not in live]
                if not free:
                    raise ValueError(f"stream models '{name}': more than {st['capacity']} distinct models in use "
                                     "(stream_model_capacity)")
                slot = free[0]
                ctx.load_bank_head(st["bank"], slot, _weights.pack_head_blob(head))
        ctx.assign_bank_head(st["bank"], None if ids.size == B else ids, np.full(ids.size, slot, np.int32))
        slots[ids] = slot
        for b in ids:
            keys[b] = key
        ctx.set_head_bank_clip_slot(st["bank"], int(slots[0]))

    def _bank_predict(self, name, n_in, n_out, x):
        """model_prediction_function of stream models: stream 0's model (zeros without one)."""
        torch = _torch()
        st = self._sbanks[name]
        x = np.ascontiguousarray(np.asarray(x, np.float32).reshape(-1, n_in, 96))
        slot = -1 if st["slots"] is None else int(st["slots"][0])
        if slot < 0:
            return [np.zeros((x.shape[0], n_out), np.float32)]
        dev = f"cuda:{self.preprocessor.device_index}"
        d = torch.from_numpy(x).to(dev)
        out = torch.empty((x.shape[0], n_out), dtype=torch.float32, device=dev)
        self.preprocessor.ctx.bank_head_predict(st["bank"], slot, d, x.shape[0], out, torch.cuda.current_stream(d.device).cuda_stream)
        return [out.cpu().numpy()]

    # ---- custom verifier models on the device (include/owwb200.h, oww_add_verifier_bank) ----
    @property
    def custom_verifier_threshold(self):
        return self._verifier_threshold

    @custom_verifier_threshold.setter
    def custom_verifier_threshold(self, value):
        """applies to the device banks from the next call on, as to the host loop"""
        self._verifier_threshold = value
        for st in list(self._vbanks.values()) + list(self._svbanks.values()):
            self.preprocessor.ctx.set_verifier_threshold(st["bank"], value)

    def _device_params(self, name, verifier):
        """(mean, weight, bias) when `verifier` is the reference's linear pipeline on `name`'s input window, else None."""
        params = linear_verifier_params(verifier)
        if params is None or params[0].size != self.model_inputs[name] * 96:
            return None
        return params

    def set_custom_verifier(self, name, verifier, streams=None):
        """Attach, replace or remove (``verifier=None``) the custom verifier of model `name` on `streams` (stream ids;
        None = every stream) from the next call on.  `verifier`: a pickle path or a loaded pipeline of the form
        ``custom_verifier_model.train_verifier_model`` produces (FunctionTransformer(flatten_features) ->
        StandardScaler -> binary LogisticRegression); anything else raises ValueError.  It runs on the device for those
        streams and replaces any host-side verifier of `name`; ``verifier=None`` on every stream also removes a host-side
        one.  ``predict_clips`` applies stream 0's verifier.  ``custom_verifier_models[name]`` follows: the verifier when
        every stream has the same one, {stream id: verifier} otherwise, absent when no stream has one."""
        if name not in self.models:
            raise ValueError(f"no model named '{name}'")
        if name in self._sbanks:
            raise ValueError(f"custom verifier models apply to wakeword_models, not to the stream models '{name}'")
        self._set_device_verifier(name, verifier, streams, False)

    def set_stream_verifier(self, name, verifier, streams=None):
        """Attach, replace or remove (``verifier=None``) the verifier of stream models `name` on `streams` (stream ids;
        None = every stream) from the next call on: where a stream's score is >= custom_verifier_threshold, p of its
        verifier on the newest window replaces it.  A stream without a model (slot -1 of the bank) is never verified and
        stays 0.0.  `verifier`: a pickle path or pipeline of train_verifier_model's form on the model's input window;
        anything else raises ValueError.  Slots are shared and freed as in ``set_custom_verifier``, and
        ``stream_verifiers[name]`` follows as ``custom_verifier_models[name]`` does there."""
        if name not in self._sbanks:
            raise ValueError(f"no stream models named '{name}'")
        self._set_device_verifier(name, verifier, streams, True)

    def _new_vbank(self, name, stream_model):
        pre, B = self.preprocessor, self.n_streams
        pre._ensure_streams()
        pre._verifier_banks = True
        thr = self.custom_verifier_threshold
        bank = (pre.ctx.add_bank_verifier_bank(self._sbanks[name]["bank"], B, thr) if stream_model
                else pre.ctx.add_verifier_bank(self._head_ids[name], B, thr))
        st = {"bank": bank, "slots": np.full(B, -1, np.int32), "objs": [None] * B}
        (self._svbanks if stream_model else self._vbanks)[name] = st
        return st

    def _set_device_verifier(self, name, verifier, streams, stream_model):
        B = self.n_streams
        ids = np.arange(B) if streams is None else np.unique(np.asarray(streams, np.int64).ravel())
        if ids.size == 0:
            return
        if ids.min() < 0 or ids.max() >= B:
            raise ValueError(f"stream ids must lie in [0, {B})")
        ctx = self.preprocessor.ctx
        st = (self._svbanks if stream_model else self._vbanks).get(name)
        params = None
        if verifier is not None:
            v = load_verifier(verifier) if isinstance(verifier, (str, os.PathLike)) else verifier
            params = self._device_params(name, v)
            if params is None:
                raise ValueError(f"model '{name}': only the linear verifier pipeline of train_verifier_model, on the "
                                 f"model's {self.model_inputs[name]}-row input window, runs on the device")
        if st is None:
            if params is None:
                if not stream_model and ids.size == B and self._host_verifiers.pop(name, None) is not None:
                    self.custom_verifier_models.pop(name, None)
                return
            st = self._new_vbank(name, stream_model)
        slot = -1
        if params is not None:           # a slot no other stream uses (one always exists: capacity = n_streams)
            others = np.ones(B, bool)
            others[ids] = False
            used = set(st["slots"][others].tolist())
            slot = next(k for k in range(B) if k not in used)
            ctx.load_verifier(st["bank"], slot, *params)
        ctx.assign_verifier(st["bank"], None if ids.size == B else ids, np.full(ids.size, slot, np.int32))
        st["slots"][ids] = slot
        for b in ids:
            st["objs"][b] = v if params is not None else None
        self._verifier_bookkeeping(name, stream_model)

    def _verifier_bookkeeping(self, name, stream_model=False):
        st = (self._svbanks if stream_model else self._vbanks)[name]
        attr = self.stream_verifiers if stream_model else self.custom_verifier_models
        self.preprocessor.ctx.set_verifier_clip_slot(st["bank"], int(st["slots"][0]))
        if not stream_model:
            self._host_verifiers.pop(name, None)
        objs = st["objs"]
        if all(o is None for o in objs):
            attr.pop(name, None)
        elif all(o is objs[0] for o in objs):
            attr[name] = objs[0]
        else:
            attr[name] = {b: o for b, o in enumerate(objs) if o is not None}

    def train_custom_verifiers(self, name, enrollments, N=5, threshold=0.5):
        """Train and attach a speaker verifier of model `name` for many streams at once.  enrollments: {stream id:
        (positive clips, negative clips)}, clips as WAV paths or int16 arrays.  Each user's verifier equals what
        ``custom_verifier_model.train_custom_verifier`` trains for that user alone on a Model of this configuration and
        feature_init, bit for bit, when the NumPy global RNG is in the same state before that user's offset draws
        (users draw in the order of `enrollments`; a Model without feature_init first draws one, as a fresh reference
        Model does).  The capture runs on the bulk path with the verifier banks off, so a Model that already verifies
        `name` captures the unverified scores.  Fitted verifiers (status 0 or 1) are loaded into `name`'s bank with
        oww_load_verifiers and assigned to their streams; other streams, and streams whose fit failed, keep what they
        had.  Returns {stream id: (pipeline or None, status)} (statuses of include/owwb200.h, oww_fit_verifiers).  N and
        threshold are the reference's positive-pass settings; only N=5 and threshold=0.5 are supported."""
        if name not in self.models:
            raise ValueError(f"no model named '{name}'")
        if name in self._sbanks:
            raise ValueError(f"custom verifier models apply to wakeword_models, not to the stream models '{name}'")
        return self._train_verifiers(name, enrollments, N, threshold, False)

    def train_stream_verifiers(self, name, enrollments, N=5, threshold=0.5):
        """``train_custom_verifiers`` for stream models `name`: each user's capture clip is scored by the model of that
        user's stream, and the fitted verifiers go to `name`'s stream verifiers (``set_stream_verifier``).  A stream
        without a model raises ValueError, as do multi-output models."""
        if name not in self._sbanks:
            raise ValueError(f"no stream models named '{name}'")
        return self._train_verifiers(name, enrollments, N, threshold, True)

    def _train_verifiers(self, name, enrollments, N, threshold, stream_model):
        from .custom_verifier_model import enroll
        if self.model_outputs[name] != 1:
            raise ValueError(f"model '{name}' has {self.model_outputs[name]} outputs; verifiers are trained on binary models")
        if self.speex_ns is not None:
            raise ValueError("train_custom_verifiers does not run with Speex noise suppression")
        if N != 5 or threshold != 0.5:
            raise ValueError("train_custom_verifiers captures as train_custom_verifier does: N=5, threshold=0.5")
        ids = np.array([int(b) for b in enrollments], np.int64)
        if ids.size == 0:
            return {}
        if ids.min() < 0 or ids.max() >= self.n_streams:
            raise ValueError(f"stream ids must lie in [0, {self.n_streams})")
        if stream_model:
            slots = self._sbanks[name]["slots"]
            bare = ids if slots is None else ids[slots[ids] < 0]
            if bare.size:
                raise ValueError(f"stream models '{name}': streams {bare.tolist()} have no model to enroll against")
        read = lambda c: _read_wav(c) if isinstance(c, (str, os.PathLike)) else np.asarray(c, np.int16)   # noqa: E731
        users = [([read(c) for c in pos], [read(c) for c in neg]) for pos, neg in enrollments.values()]
        pre, ctx = self.preprocessor, self.preprocessor.ctx
        fi = pre._feature_init
        if fi is None:
            fi = pre._get_embeddings(np.random.randint(-1000, 1000, 16000 * 4).astype(np.int16))
        banks = self._vbanks or self._svbanks
        if banks:
            ctx.enable_verifiers(False)
        try:
            res = enroll(self, name, users, feature_init=fi, streams=ids if stream_model else None)
        finally:
            if banks:
                ctx.enable_verifiers(True)
        ok = [i for i, r in enumerate(res) if r["status"] in (0, 1)]
        if ok:
            torch = _torch()
            B = self.n_streams
            st = (self._svbanks if stream_model else self._vbanks).get(name)
            if st is None:
                st = self._new_vbank(name, stream_model)
            sid = ids[ok]
            others = np.ones(B, bool)
            others[sid] = False
            used = set(st["slots"][others].tolist())
            slots = np.array([k for k in range(B) if k not in used][:sid.size], np.int32)
            dev = torch.device("cuda", pre.device_index)
            t = lambda key: torch.from_numpy(np.stack([res[i][key] for i in ok])).to(dev)   # noqa: E731
            ctx.load_verifiers(st["bank"], slots, t("mean"), t("weight"), t("bias"),
                               torch.cuda.current_stream(dev).cuda_stream)
            ctx.assign_verifier(st["bank"], sid, slots, torch.cuda.current_stream(dev).cuda_stream)
            st["slots"][sid] = slots
            for i, b in zip(ok, sid):
                st["objs"][b] = res[i]["pipeline"]
            self._verifier_bookkeeping(name, stream_model)
        return {int(b): (r["pipeline"], r["status"]) for b, r in zip(ids, res)}

    def _reverify(self, mdl, predictions, labels, streams):
        """Verification on the host side of the stateless entry, on each stream's newest window (model.py:319-328): for
        calls that run no step (< 1280 samples: the previous prediction is re-verified, as the reference does) and for
        calls split into several device steps (> max_chunks chunks: those run without the banks, and the max over all
        their chunk windows is verified here, once).  Of `streams` (bool [B]): those with a device verifier and a label >=
        the threshold."""
        st = self._vbanks.get(mdl) or self._svbanks[mdl]
        thr = np.float32(self.custom_verifier_threshold)
        hit = np.zeros(self.n_streams, bool)
        for lab in labels:
            hit |= predictions[lab] >= thr
        hit &= (st["slots"] >= 0) & streams & self._has_model(mdl, np.arange(self.n_streams))
        for slot in np.unique(st["slots"][hit]):
            bs = np.nonzero(hit & (st["slots"] == slot))[0]
            feats = np.concatenate([self.preprocessor.get_features(self.model_inputs[mdl], stream=int(b)) for b in bs])
            p = self.preprocessor.ctx.verifier_predict_host(st["bank"], int(slot), feats)
            for lab in labels:
                sel = predictions[lab][bs] >= thr
                predictions[lab][bs[sel]] = p[sel]

    def _has_model(self, mdl, streams):
        """bool per stream id: `mdl` scores it (always, but for stream models on slot -1: never verified)"""
        sb = self._sbanks.get(mdl)
        if sb is None:
            return np.ones(len(streams), bool)
        return np.zeros(len(streams), bool) if sb["slots"] is None else sb["slots"][streams] >= 0

    # ---- per-label history (model.py:198; vectorised over streams) ----
    def _reset_history(self):
        self._hist = {}        # label -> float32 [30, B] ring of the last predictions
        self._count = {}       # label -> int64 [B] predictions appended so far
        # True once detect* has run: the device detector then holds the history, and _hist / _count are refreshed from
        # it where they are read (_pull_history); the next predict* takes it back
        self._hist_on_device = False

    def _pull_history(self):
        """_hist / _count <- the device detector's history, while it is the one in use"""
        if not self._hist_on_device:
            return
        hist, cnt = self.preprocessor.ctx.detector_history(np.arange(self.n_streams, dtype=np.int32))
        cnt = cnt.astype(np.int64)
        slot = (np.arange(30)[:, None] - cnt[None, :]) % 30       # ring slot s holds the entry (s - count) % 30 of oldest-first
        for j, lab in enumerate(self.labels()):
            h, c = self._h(lab)
            h[:] = hist[:, j, :].T[slot, np.arange(self.n_streams)[None, :]]
            c[:] = cnt

    def _push_history(self, ids):
        """the device detector's history of streams ids <- _hist / _count"""
        ids = np.asarray(ids, np.int64)
        labels = self.labels()
        hist = np.zeros((ids.size, len(labels), 30), np.float32)
        cnt = self._h(labels[0])[1][ids]
        for j, lab in enumerate(labels):
            hist[:, j, :] = self._recent(lab, 30)[0][:, ids].T
        self.preprocessor.ctx.set_detector_history(ids.astype(np.int32), hist, np.minimum(cnt, 2 ** 30).astype(np.int32))

    def _h(self, label):
        if label not in self._hist:
            self._hist[label] = np.zeros((30, self.n_streams), np.float32)
            self._count[label] = np.zeros(self.n_streams, np.int64)
        return self._hist[label], self._count[label]

    def _recent(self, label, n):
        """Per stream its own last min(n_b, count_b, 30) appended predictions (deque(maxlen=30) view): -> (float32
        [30, B] each stream's history oldest first, bool [30, B] which entries are among those).  n: int or int [B]."""
        hist, cnt = self._h(label)
        i = np.arange(30)[:, None]
        ordered = hist[(cnt[None, :] - 30 + i) % 30, np.arange(self.n_streams)[None, :]]
        k = np.minimum(np.minimum(np.asarray(n, np.int64), cnt), 30)
        return ordered, i >= 30 - k[None, :]

    @property
    def prediction_buffer(self):
        """defaultdict(deque(maxlen=30)) of stream 0's history, like the reference attribute."""
        self._pull_history()
        buf = defaultdict(partial(deque, maxlen=30))
        for label in self._hist:
            ordered, valid = self._recent(label, 30)
            for v in ordered[valid[:, 0], 0]:
                buf[label].append(float(v))
        return buf

    def reset_streams(self, stream_ids, feature_init=None):
        """Reset the listed streams only: device state, samples not yet stepped and prediction history (a new client on
        a stream gets the first-5 zeroing of model.py:330-333 again).  The other streams are untouched."""
        ids = np.asarray(stream_ids, np.int64).ravel()
        if ids.size and (ids.min() < 0 or ids.max() >= self.n_streams):
            raise ValueError(f"stream ids must be in [0, {self.n_streams})")
        self.preprocessor.reset(feature_init, stream_ids=ids.astype(np.int32))
        for label in self._hist:
            self._hist[label][:, ids] = 0.0
            self._count[label][ids] = 0

    # ---- moving live streams (include/owwb200.h, oww_export_streams) ----
    def export_streams(self, stream_ids):
        """-> StreamState of the listed streams: their device state, the samples they hold not yet stepped and their
        prediction history.  ``import_streams`` on a Model of the same configuration continues them exactly."""
        ids = self._ids(stream_ids)
        pre = self.preprocessor
        pre._ensure_streams()
        _, key = pre.ctx.stream_state_info()
        records = pre.ctx.export_records(ids)
        buf, lens = pre._ragged_pending()
        labels = self.labels()
        self._pull_history()
        audio = None
        if pre.audio_history_samples:
            audio = pre.ctx.audio_state(ids) + (pre._held_in_raw[ids].copy(),)
        ingest = pre.ctx.ingest_state(ids) if pre.ingest else None
        return StreamState(records, key, labels, [buf[b, :lens[b]].copy() for b in ids],
                           {lab: self._h(lab)[0][:, ids].copy() for lab in labels},
                           {lab: self._h(lab)[1][ids].copy() for lab in labels}, audio, ingest,
                           [self._stream_det.get(b) for b in ids.tolist()])

    def import_streams(self, stream_ids, state):
        """Streams stream_ids (distinct) become the streams `state` was exported from: device state, samples not yet
        stepped, prediction history (first-5 zeroing, patience, debounce) and detection settings (set_stream_detection;
        none when the state has none).  Their stream models and verifiers stay as
        they are here.  ValueError: another configuration (cnn_mode, split_from, weights), another label set, or Speex
        noise suppression on (its state cannot be exported)."""
        ids = self._ids(stream_ids)
        if self.speex_ns:
            raise ValueError("streams cannot be imported with Speex noise suppression on: its state is not exported")
        if ids.size != len(state):
            raise ValueError(f"{ids.size} stream ids for {len(state)} exported streams")
        if len(set(ids.tolist())) != ids.size:
            raise ValueError("stream ids must be distinct")
        pre = self.preprocessor
        pre._ensure_streams()
        if state.key != pre.ctx.stream_state_info()[1]:
            raise ValueError("the streams were exported under another configuration (cnn_mode, split_from or weights)")
        if list(state.labels) != self.labels():
            raise ValueError(f"the streams were exported with the labels {list(state.labels)}, this Model has {self.labels()}")
        h_state = 0 if state.audio is None else state.audio[0].shape[1]
        if h_state != pre.audio_history_samples:
            raise ValueError(f"the streams were exported with an audio history of {h_state} samples, this Model keeps "
                             f"{pre.audio_history_samples}")
        if (state.ingest is not None) != pre.ingest:
            raise ValueError("the streams were exported from a Model " + ("with" if state.ingest is not None else "without")
                             + " device ingest (sr=...), this Model " + ("has it" if pre.ingest else "has not"))
        if self.speex_ns is not None and state.ingest is not None and (state.ingest[0] != 16000).any():
            self._check_speex_rates(state.ingest[0])
        pre.ctx.import_records(ids, state.records)
        if state.ingest is not None:
            pre.ctx.set_ingest_state(ids, *state.ingest)
            pre.sample_rates[ids] = state.ingest[0]
        if state.audio is not None:
            pre.ctx.set_audio_state(ids, state.audio[0], state.audio[1])
            pre._held_in_raw[ids] = state.audio[2]
        buf, lens = pre._ragged_pending()
        for i, b in enumerate(ids):
            p = state.pending[i]
            buf[b] = 0
            buf[b, :p.size] = p
            lens[b] = p.size
        pre._set_ragged_pending(buf, lens)
        for lab in state.labels:
            hist, cnt = self._h(lab)
            hist[:, ids] = state.history[lab]
            cnt[ids] = state.counts[lab]
        if self._hist_on_device and ids.size:
            self._push_history(ids)
        for i, b in enumerate(ids.tolist()):
            if state.detection is None or state.detection[i] is None:
                self._stream_det.pop(b, None)
            else:
                self._stream_det[b] = state.detection[i]
        self._stream_det_pushed = False

    def _ids(self, stream_ids):
        ids = np.asarray(stream_ids, np.int64).ravel()
        if ids.size and (ids.min() < 0 or ids.max() >= self.n_streams):
            raise ValueError(f"stream ids must be in [0, {self.n_streams})")
        return ids.astype(np.int32)

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

    # ---- audio at other sample rates (AudioFeatures(sr=...), include/owwb200.h, oww_ingest) ----
    def set_sample_rates(self, stream_ids, rates):
        """Streams stream_ids take audio at rates[i] (one int for all, or one per id; a rate of the library's table) from
        the next call on; their resamplers restart, the 16 kHz samples they hold are kept.  ValueError on a Model built
        without device ingest (sr=16000, the default)."""
        if not self.preprocessor.ingest:
            raise ValueError("set_sample_rates needs device ingest: construct the Model with sr=<rate> or "
                             "sr=[one rate per stream]")
        if self.speex_ns is not None and (np.asarray(rates) != 16000).any():
            self._check_speex_rates(np.asarray(rates))
        self.preprocessor.set_sample_rates(stream_ids, rates)

    def _check_speex_rates(self, rates=None):
        pre = self.preprocessor
        rates = pre.sample_rates if rates is None else rates
        if self.speex_ns is not None and pre.ingest and (rates != 16000).any():
            raise ValueError("Speex noise suppression runs on 16 kHz audio only; it cannot be combined with streams at "
                             "other sample rates")

    def _no_ingest(self, what, hint=""):
        if self.preprocessor.ingest:
            raise ValueError(f"{what} takes 16 kHz clips; this Model takes streams at other sample rates (sr=...)"
                             + hint)

    def _clip_rates(self, sr, n, what):
        """sr of a clip call (None, one rate, or one per clip) -> int32 [n] rates, or None when the clips are 16 kHz
        (no sr on a Model without device ingest, or every rate 16000).  No sr on a device-ingest Model raises."""
        if sr is None:
            self._no_ingest(what, "; pass the clips' rates as sr=")
            return None
        rates = np.asarray(sr, np.int64).ravel()
        if rates.size not in (1, n):
            raise ValueError(f"sr has {rates.size} rates for {n} clips")
        for r in np.unique(rates):
            _native.resampler_taps(int(r))                   # ValueError outside the table
        rates = np.ascontiguousarray(np.broadcast_to(rates, (n,)), np.int32)
        return None if (rates == 16000).all() else rates

    def _suppress_noise_with_speex(self, x, frame_size=160):
        cleaned = [self.speex_ns.process(x[i:i + frame_size].tobytes()) for i in range(0, x.shape[0], frame_size)]
        return np.frombuffer(b"".join(cleaned), np.int16)

    def predict(self, x, patience={}, threshold={}, debounce_time=0.0, timing=False):
        """One streaming step (model.py:232-386).  x: ndarray [samples] (n_streams == 1) or
        [n_streams, samples].  Returns {label: float} for a single stream, {label: float32[B]} otherwise."""
        if not isinstance(x, np.ndarray):
            raise ValueError(f"The input audio data (x) must by a Numpy array, instead received an object of type {type(x)}.")
        single = self.n_streams == 1
        t0 = time.time()
        if self.speex_ns:
            if not single:
                raise ValueError("Speex noise suppression is single-stream")
            x = self._suppress_noise_with_speex(x)
        if self.preprocessor.pending_ragged:
            # the streams hold different remainders (after predict_ragged / reset_streams): per-stream accumulation
            n_prepared, n_chunks, split = self.preprocessor._streaming_features_ragged(list(self.preprocessor._coerce(x)),
                                                                                       self._scores)
        else:
            n_prepared, n_chunks = self.preprocessor._streaming_features(x, self._scores)
            split = n_chunks > self.preprocessor.max_chunks
            n_prepared = np.full(self.n_streams, n_prepared, np.int64)
        return self._finish(n_prepared, split, patience, threshold, debounce_time, timing, t0, single)

    def predict_ragged(self, x, patience={}, threshold={}, debounce_time=0.0, timing=False):
        """One streaming step in which every stream gets its own samples: x is a sequence of n_streams 1-D NumPy arrays of
        any lengths (0 included).  Stream b's result, state and history are those of an independent reference
        ``Model`` that was given the same arrays: it steps the whole chunks of its own remainder + x[b] and keeps the
        rest; with fewer than 1280 samples prepared it returns its previous prediction (one-output heads) or zeros, and
        first-5 zeroing, patience and debounce use its own history and sample count.  A stream with no samples prepared
        at all (n_prepared == 0) has a debounce window of its whole 30-entry history, the limit of the reference's
        formula (which divides by zero there).  Returns {label: float32[B]} (a float per label for one stream)."""
        B = self.n_streams
        try:
            n = len(x)
        except TypeError:
            raise ValueError(f"predict_ragged takes a sequence of {B} 1-D NumPy arrays, got {type(x)}") from None
        if n != B:
            raise ValueError(f"predict_ragged takes one array per stream ({B}), got {n}")
        xs = []
        for b, a in enumerate(x):
            if not isinstance(a, np.ndarray):
                raise ValueError(f"The input audio data (x[{b}]) must by a Numpy array, instead received an object of "
                                 f"type {type(a)}.")
            if a.ndim != 1:
                raise ValueError(f"x[{b}] must be 1-D, got shape {a.shape}")
            xs.append(a if a.dtype == np.int16 else a.astype(np.int16))
        t0 = time.time()
        if self.speex_ns:
            if B != 1:
                raise ValueError("Speex noise suppression is single-stream")
            xs = [self._suppress_noise_with_speex(xs[0])]
        n_prepared, _, split = self.preprocessor._streaming_features_ragged(xs, self._scores)
        return self._finish(n_prepared, split, patience, threshold, debounce_time, timing, t0, B == 1)

    # ---- detections on the device (include/owwb200.h, oww_set_detector / oww_detect) ----
    def detect(self, x, threshold, patience={}, debounce_time=0.0, capture=None):
        """``predict(x, patience, threshold, debounce_time)`` that returns only the detections of this call: a list of
        (stream id, label, score) for every label whose prediction is >= the threshold of its model, ordered by stream,
        then by label in ``labels()`` order.  threshold: {model name: float} as in the reference (a model without one
        never fires), or one float for every model.  State and history advance exactly as in ``predict``; the history,
        the first-5 zeroing, patience and debounce run on the device (csrc/detect.cu), the scores stay there, and only
        the event count and the events are copied back.  ``predict*`` and ``detect*`` may be mixed freely: the history
        moves between host and device at each switch (one copy of [n_streams, labels, 30] floats), and
        ``prediction_buffer``, ``reset``, ``reset_streams``, ``export_streams`` and ``import_streams`` see it wherever it is.
        Streams given settings of their own (``set_stream_detection``) detect with those in place of the call's.

        ValueError, so that no call needs per-stream host work: a custom verifier that only runs on the host; Speex noise
        suppression with more than one stream; a stream that prepares more than ``max_chunks`` chunks in one call while
        device verifier banks are loaded (``predict`` re-verifies that case on the host).

        One difference from ``predict``, only on models with device verifier banks: a stream that prepares fewer than
        1280 samples repeats its previous prediction as stored; ``predict`` passes the repeated value through the
        verifier once more.

        capture: seconds (needs ``audio_history``).  Each event then becomes (stream id, label, score, audio, end): audio
        = the last ``capture`` seconds the stream stepped (int16; zeros for what its history does not hold), gathered on
        the device right after the detection, and end = the stream's sample position at its last sample (what
        ``get_audio(end=...)`` takes for audio after the event).  Without capture the return value is unchanged."""
        if not isinstance(x, np.ndarray):
            raise ValueError(f"The input audio data (x) must by a Numpy array, instead received an object of type {type(x)}.")
        self._detect_refusals()
        if self.speex_ns:
            x = self._suppress_noise_with_speex(x)
        return self._detect(self.preprocessor._coerce(x), threshold, patience, debounce_time, capture)

    def detect_ragged(self, x, threshold, patience={}, debounce_time=0.0, capture=None):
        """``detect`` with the inputs of ``predict_ragged``: one 1-D array of any length per stream."""
        B = self.n_streams
        try:
            n = len(x)
        except TypeError:
            raise ValueError(f"detect_ragged takes a sequence of {B} 1-D NumPy arrays, got {type(x)}") from None
        if n != B:
            raise ValueError(f"detect_ragged takes one array per stream ({B}), got {n}")
        xs = []
        for b, a in enumerate(x):
            if not isinstance(a, np.ndarray) or a.ndim != 1:
                raise ValueError(f"x[{b}] must be a 1-D NumPy array")
            xs.append(a if a.dtype == np.int16 else a.astype(np.int16))
        self._detect_refusals()
        if self.speex_ns:
            xs = [self._suppress_noise_with_speex(xs[0])]
        return self._detect(xs, threshold, patience, debounce_time, capture)

    def _detect_refusals(self):
        if self._host_verifiers:
            raise ValueError(f"detect: the custom verifiers of {sorted(self._host_verifiers)} run on the host only (only "
                             "the linear pipeline of train_verifier_model runs on the device); use predict")
        if self.speex_ns and self.n_streams != 1:
            raise ValueError("Speex noise suppression is single-stream")

    def _detector_table(self, threshold, patience, debounce_time):
        """-> [(column, repeats, threshold or None, patience)] per label of labels(), as predict applies its arguments"""
        if patience != {} and debounce_time > 0:
            raise ValueError("Error! The `patience` and `debounce_time` arguments cannot be used together!")
        table = []
        for mdl in self.models:
            col0, n_out = self._columns[mdl]
            if n_out == 1:
                entries = [(mdl, col0, True)]
            else:
                entries = [(cls, col0 + int(k) if int(k) < n_out else -1, False) for k, cls in self.class_mapping[mdl].items()]
            for lab, col, repeats in entries:
                parent = self.get_parent_model_from_label(lab)
                thr = threshold.get(parent) if isinstance(threshold, dict) else threshold
                pat = int(patience.get(parent, 0))
                if pat and thr is None:
                    raise ValueError("Error! When using the `patience` argument, threshold "
                                     "values must be provided via the `threshold` argument!")
                if not 0 <= pat <= 30:
                    raise ValueError(f"patience of '{parent}' must lie in 0..30 (the history holds 30 predictions)")
                table.append((col, repeats, None if thr is None else float(thr), pat))
        return table

    # ---- per-stream detection settings (include/owwb200.h, oww_set_stream_detection) ----
    def set_stream_detection(self, stream_ids, threshold=None, patience=None, debounce_time=None):
        """Streams stream_ids detect at their own sensitivity in ``detect`` / ``detect_ragged``: threshold - one float for
        every model, or {model name: float, or None for no threshold on these streams}; patience - {model name: 0..30};
        debounce_time - seconds.  Each given value replaces, on these streams, the one the ``detect*`` call passes; what
        is not given (None, a model missing from a dict) stays the call's.  Names resolve as in ``predict`` (a multi-class
        model's labels take its values; stream models by their name).  The call replaces the streams' earlier settings.
        ``predict*`` keep taking their per-call arguments only.  Each stream's resulting settings are checked at the next
        ``detect*`` as ``predict`` checks its arguments (ValueError before anything runs).  ``reset*`` keep the settings;
        ``export_streams`` / ``import_streams`` move them with the streams."""
        ids = self._ids(stream_ids)
        if isinstance(threshold, dict):
            threshold = {k: None if v is None else float(v) for k, v in threshold.items()}
        elif threshold is not None:
            threshold = float(threshold)
        patience = {k: int(v) for k, v in (patience or {}).items()}
        for name in list(threshold if isinstance(threshold, dict) else []) + list(patience):
            if name not in self.models:
                raise ValueError(f"no model named '{name}'; the models are {list(self.models)}")
        for name, pat in patience.items():
            if not 0 <= pat <= 30:
                raise ValueError(f"patience of '{name}' must lie in 0..30 (the history holds 30 predictions)")
        if debounce_time is not None:
            debounce_time = float(debounce_time)
            if not debounce_time >= 0 or not np.isfinite(debounce_time):
                raise ValueError("debounce_time must be finite and >= 0")
            if patience and debounce_time > 0:
                raise ValueError("Error! The `patience` and `debounce_time` arguments cannot be used together!")
        for b in ids.tolist():
            self._stream_det[b] = (threshold, patience, debounce_time)
        self._stream_det_pushed = False

    def clear_stream_detection(self, stream_ids=None):
        """Streams stream_ids (None = all) detect with the settings of each ``detect*`` call again."""
        for b in (range(self.n_streams) if stream_ids is None else self._ids(stream_ids).tolist()):
            self._stream_det.pop(b, None)
        self._stream_det_pushed = False

    def stream_detection(self, stream_id):
        """-> {"threshold", "patience", "debounce_time"} as set_stream_detection took them for the stream, or None"""
        s = self._stream_det.get(int(stream_id))
        return None if s is None else dict(threshold=s[0], patience=dict(s[1]), debounce_time=s[2])

    def _stream_detection_table(self, threshold, patience, debounce_time):
        """-> None when no stream has settings of its own, else (STREAM_DETECT_DTYPE [n_streams, labels], float64
        [n_streams] debounce): each such stream's settings over the call's, resolved by _detector_table (and checked
        there), the others the handle's.  Streams with the same settings are resolved once."""
        if not self._stream_det:
            return None
        rec = np.zeros((self.n_streams, len(self.labels())), _native.STREAM_DETECT_DTYPE)
        rec["threshold"], rec["patience"] = np.nan, -1
        deb = np.full(self.n_streams, np.nan)
        groups = {}
        for b, (thr, pat, dt) in self._stream_det.items():
            key = (tuple(sorted(thr.items())) if isinstance(thr, dict) else thr, tuple(sorted(pat.items())), dt)
            groups.setdefault(key, ([], (thr, pat, dt)))[0].append(b)
        for ids, (thr, pat, dt) in groups.values():
            if thr is None:
                thr = threshold
            elif isinstance(thr, dict):
                thr = {**(threshold if isinstance(threshold, dict) else {m: threshold for m in self.models}), **thr}
            dt = debounce_time if dt is None else dt
            rows = self._detector_table(thr, {**patience, **pat}, dt)
            ids = np.asarray(ids)
            for j, (_, _, t, p) in enumerate(rows):
                rec["threshold"][ids, j] = np.nan if t is None else t
                rec["flags"][ids, j] = _native.DETECT_NO_THRESHOLD if t is None else 0
                rec["patience"][ids, j] = p
            deb[ids] = dt
        return rec, deb

    def _detect(self, xs, threshold, patience, debounce_time, capture=None):
        pre = self.preprocessor
        pre._ensure_streams()
        ctx = pre.ctx
        labels = self.labels()
        if not labels:
            raise ValueError("detect needs at least one model")
        n_capture = None if capture is None else self._audio_samples(capture)
        table = self._detector_table(threshold, patience, debounce_time)
        lockstep = isinstance(xs, np.ndarray) and not pre.pending_ragged      # as predict: one length, one remainder
        if not lockstep:
            xs = list(xs)
        n_in = np.array([a.shape[0] for a in xs], np.int64)
        if pre.ingest:                  # more than one ingest call
            too_long = (self._vbanks or self._svbanks) and (n_in > ctx.ingest_capacity()).any()
        else:
            held = pre._pending.shape[1] if not pre.pending_ragged else pre._ragged_pending()[1]
            too_long = (self._vbanks or self._svbanks) and ((held + n_in) // CHUNK > pre.max_chunks).any()
        if too_long:
            raise ValueError(f"detect: a stream prepares more than max_chunks={pre.max_chunks} chunks in this call while "
                             "custom verifiers are loaded; construct the Model with a larger max_chunks, or use predict")
        config = (table, float(debounce_time))
        call = (repr(threshold), repr(patience), float(debounce_time))
        if self._stream_det_pushed != call:                        # checks every stream's settings before any change
            stream_table = self._stream_detection_table(threshold, patience, debounce_time)
        if getattr(self, "_detector_config", None) != config:      # oww_set_detector synchronises: only on a change
            ctx.set_detector(table, debounce_time)                  # ... and clears every stream's settings
            self._detector_config = config
            self._stream_det_on_device = False
        if self._stream_det_pushed != call:
            if stream_table is not None or self._stream_det_on_device:
                ctx.set_stream_detection(None, *(stream_table or (None, None)))
            self._stream_det_on_device = stream_table is not None
            self._stream_det_pushed = call
        if not self._hist_on_device:
            if self._hist:
                self._push_history(np.arange(self.n_streams))
            self._hist_on_device = True
        if getattr(self, "_d_scores", None) is None:
            self._d_scores = ctx.new_scores()
        if lockstep:
            n_prepared = pre._streaming_features(xs, self._d_scores, device=True)[0]
        else:
            n_prepared = pre._streaming_features_ragged(xs, self._d_scores, device=True)[0].astype(np.int32)
        if n_capture is None:
            events, n = ctx.detect_events(self._d_scores, n_prepared)
            return list(zip(events["stream"].tolist(), [labels[j] for j in events["label"].tolist()],
                            events["score"].tolist()))
        events, n, clips, ends = ctx.detect_capture(self._d_scores, n_prepared, n_capture)
        clips = clips.cpu().numpy()
        return list(zip(events["stream"].tolist(), [labels[j] for j in events["label"].tolist()], events["score"].tolist(),
                        list(clips), ends.tolist()))

    # ---- stream audio on the device (include/owwb200.h, oww_set_audio_history) ----
    def _audio_samples(self, seconds):
        H = self.preprocessor.audio_history_samples
        if not H:
            raise ValueError("stream audio needs the audio history: construct the Model with audio_history=<seconds>")
        n = int(round(float(seconds) * 16000))
        if not 1 <= n <= H:
            raise ValueError(f"{seconds} s is outside (0, {H / 16000}] s, the audio history")
        return n

    def get_audio(self, stream_ids, seconds, end=None):
        """The audio the listed streams stepped (ids may repeat) -> (int16 [n, samples], int64 [n] ends): row i = the
        ``seconds`` of stream stream_ids[i] that end at sample position end[i] (the samples the stream has stepped since
        its reset; None or < 0: its current position, which ``ends`` then reports).  Samples the history does not hold -
        before it, overwritten, or not stepped yet (an end past the position asks for audio after an event, to be read
        once the stream has advanced) - are zeros.  Samples held back because they do not fill a chunk are not
        included: only stepped audio is, addressed by stream sample position."""
        pre = self.preprocessor
        pre._ensure_streams()
        n = self._audio_samples(seconds)
        ids = self._ids(stream_ids)
        e = None if end is None else np.broadcast_to(np.asarray(end, np.int64), ids.shape).copy()
        clips, pos = pre.ctx.read_audio(ids, n, e)
        pos = pos.cpu().numpy()
        return clips.cpu().numpy(), pos if e is None else np.where(e >= 0, e, pos)

    def _finish(self, n_prepared, split, patience, threshold, debounce_time, timing, t0, single):
        """model.py:285-386 per stream after the device step(s): stream b prepared n_prepared[b] samples (its row of
        self._scores holds the step's scores when >= 1280); split: the steps ran without the verifier banks."""
        self._pull_history()                     # after detect*: the history comes back to the host
        self._hist_on_device = False
        if timing:
            timing_dict = {"models": {"preprocessor": time.time() - t0}}
        B = self.n_streams
        ar = np.arange(B)
        stepped = n_prepared >= CHUNK
        reverify = ~stepped | split
        predictions = {}
        for mdl in self.models.keys():
            if timing:
                t1 = time.time()
            col0, n_out = self._columns[mdl]
            if n_out == 1:
                hist, cnt = self._h(mdl)
                prev = np.where(cnt > 0, hist[(cnt - 1) % 30, ar], np.float32(0.0))
                pred = np.where(stepped, self._scores[:, col0], prev).astype(np.float32)[:, None]
            else:
                n_classes = max(int(i) for i in self.class_mapping[mdl].keys())
                pred = np.zeros((B, max(n_classes + 1, n_out)), np.float32)
                pred[stepped, :n_out] = self._scores[stepped, col0:col0 + n_out]   # max over chunk windows done on device
            if n_out == 1:
                predictions[mdl] = pred[:, 0].copy()
                labels = [mdl]
            else:
                labels = list(self.class_mapping[mdl].values())
                for int_label, cls in self.class_mapping[mdl].items():
                    predictions[cls] = pred[:, int(int_label)].copy()
            if (mdl in self._vbanks or mdl in self._svbanks) and reverify.any():
                self._reverify(mdl, predictions, labels, reverify)   # otherwise the device verified the step it ran

            if self._host_verifiers != {}:
                for cls in list(predictions.keys()):
                    parent = self.get_parent_model_from_label(cls)
                    if self._host_verifiers.get(parent, False):
                        for b in np.nonzero(predictions[cls] >= self.custom_verifier_threshold)[0]:
                            feats = self.preprocessor.get_features(self.model_inputs[mdl], stream=int(b))
                            predictions[cls][b] = self._host_verifiers[parent].predict_proba(feats)[0][-1]

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
                    sc, valid = self._recent(lab, patience[parent])
                    fail = ((sc >= threshold[parent]) & valid).sum(axis=0) < patience[parent]
                    predictions[lab] = np.where(nz & fail, np.float32(0.0), predictions[lab])
                elif debounce_time > 0 and parent in threshold.keys():
                    with np.errstate(divide="ignore"):
                        n_frames = np.where(n_prepared > 0, np.ceil(debounce_time / (n_prepared / 16000)), 30)
                    rec, valid = self._recent(lab, n_frames.astype(np.int64))
                    hit = ((rec >= threshold[parent]) & valid).sum(axis=0) > 0
                    predictions[lab] = np.where(nz & (predictions[lab] >= threshold[parent]) & hit,
                                                np.float32(0.0), predictions[lab])

        for lab in predictions.keys():
            hist, cnt = self._h(lab)
            hist[cnt % 30, ar] = predictions[lab]
            cnt += 1

        out = {k: (float(v[0]) if single else v) for k, v in predictions.items()}
        if timing:
            return out, timing_dict
        return out

    def predict_clip(self, clip, padding=1, chunk_size=1280, sr=None, **kwargs):
        """model.py:388-426: path or int16 array -> list of per-step dicts (no reset, like the reference).  A WAV is read
        at its header's rate (an ``sr`` that disagrees raises ValueError), an array is at ``sr`` (default 16000).  At
        another rate the clip is resampled to 16 kHz on the device with its padding, and ``chunk_size`` counts 16 kHz
        samples.  A Model with device ingest refuses whatever ``sr``: its ``predict`` takes audio at the stream's rate."""
        if isinstance(clip, str):
            data, rate = _read_wav_rate(clip)
            if sr is not None and int(sr) != rate:
                raise ValueError(f"{clip}: the header says {rate} Hz, sr={sr}")
        elif isinstance(clip, np.ndarray):
            data, rate = clip, 16000 if sr is None else int(sr)
        else:
            raise ValueError("clip must be a WAV path or a numpy array")
        if self.n_streams != 1:
            raise ValueError("predict_clip is single-stream; use predict_clips for batches")
        self._no_ingest("predict_clip")
        if rate != 16000:
            x = np.asarray(data).astype(np.int16, copy=False).ravel()
            d, _ = self.preprocessor.resample_clips(x, [0, x.size], rate, 16000 * int(padding))
            data = d.cpu().numpy()
        elif padding:
            z = np.zeros(16000 * padding).astype(np.int16)
            data = np.concatenate((z, data, z))
        return [self.predict(data[i:i + chunk_size], **kwargs) for i in range(0, data.shape[0] - chunk_size, chunk_size)]

    def _get_positive_prediction_frames(self, file, threshold=0.5, return_type="features", **kwargs):
        """model.py:428-478: run the WAV through ``predict`` in 1280-sample steps and collect, per label, what produced
        a score >= ``threshold``: the head's input features ``[n_in, 96]`` at that step (``return_type="features"``) or
        the 4 s of audio around it (``"audio"``: 3 s before, 1 s after; steps without a full 4 s are dropped).
        Returns {label: stacked array}; labels without a hit are absent.  A WAV at another rate than 16 kHz is resampled
        on the device first, and the audio context is cut from the 16 kHz samples."""
        if return_type not in ("features", "audio"):
            raise ValueError("return_type must be 'features' or 'audio'")
        if self.n_streams != 1:
            raise ValueError("_get_positive_prediction_frames is single-stream")
        self._no_ingest("_get_positive_prediction_frames")
        data, rate = _read_wav_rate(file)
        if rate != 16000:
            d, _ = self.preprocessor.resample_clips(data, [0, data.size], rate, 0)
            data = d.cpu().numpy()
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

    def predict_clips(self, clips, padding=1, feature_init=None, chunk_size=1280, streams=None, sr=None, patience={},
                      threshold={}, debounce_time=0.0):
        """Bulk path (extension; SURVEY.md F9): each clip from a fresh state, in one device call.  ``clips``: an int16
        [N,S] array or tensor, or a sequence of 1-D int16 arrays of any lengths.  Returns a list (per clip) of lists (per
        call) of {label: float}, i.e. what predict_clip(clip, padding, chunk_size, patience=patience,
        threshold=threshold, debounce_time=debounce_time) would return for each clip after reset(feature_init).  streams
        (N stream ids, or None: stream 0's models and verifiers): clip i is predicted as stream streams[i] would predict
        it, with its stream models and device verifiers.  sr: as in predict_clips_ragged.  patience, threshold,
        debounce_time: as in ``predict``, with the same ValueErrors; the history, the first-5 zeroing, patience and
        debounce run on the device (oww_detect_clips)."""
        rates = self._clip_rates(sr, len(clips), "predict_clips")
        torch = _torch()
        if rates is None and (sr is None or not self.preprocessor.ingest) and streams is None and chunk_size == CHUNK \
                and (isinstance(clips, torch.Tensor) or (isinstance(clips, np.ndarray) and clips.ndim == 2)):
            scores, labels = self.predict_clips_array(clips, padding, feature_init, patience, threshold, debounce_time)
            return [[{lab: float(scores[c, s, j]) for j, lab in enumerate(labels)} for s in range(scores.shape[1])]
                    for c in range(scores.shape[0])]
        pcm, offsets = _concat_clips(clips)
        scores, row_off, labels = self.predict_clips_ragged(pcm, offsets, padding, chunk_size, feature_init, streams,
                                                            sr=sr, patience=patience, threshold=threshold,
                                                            debounce_time=debounce_time)
        return _rows_to_dicts(scores, row_off, labels)

    def predict_clips_ragged(self, pcm, offsets, padding=1, chunk_size=1280, feature_init=None, streams=None, sr=None,
                             patience={}, threshold={}, debounce_time=0.0):
        """Array form of the bulk path over clips of any lengths: clip i is ``pcm[offsets[i]:offsets[i+1]]`` (int16 1-D
        array or tensor, int64 offsets).  Returns (float32 [rows, n_labels], int64 row_offsets [N+1], labels): clip i's
        rows ``row_offsets[i]:row_offsets[i+1]`` are the predictions predict_clip(clip, padding, chunk_size, patience=...,
        threshold=..., debounce_time=...) returns after reset(feature_init), one per call.  streams, patience,
        threshold, debounce_time: as in predict_clips.  sr: the clips' rate, one for all or one per clip (None: 16 kHz).
        Clips at other rates are resampled to 16 kHz with their padding in one device launch
        (AudioFeatures.resample_clips) and then run as 16 kHz clips without padding: ``chunk_size`` counts 16 kHz samples
        and a clip makes len(range(0, L - chunk_size, chunk_size)) calls over its L = A(S) + 2*16000*padding samples."""
        table = self._clip_table(patience, threshold, debounce_time)
        rules = dict(table=table, debounce_time=debounce_time) if patience or threshold or debounce_time > 0 else {}
        pcm, offsets, padding, check = self._clips_16k(pcm, offsets, padding, sr)
        return self._predict_ragged(pcm, offsets, padding, chunk_size, feature_init, streams=streams, check_ingest=check,
                                    **rules)[:3]

    def detect_clips(self, clips, threshold, patience={}, debounce_time=0.0, padding=1, chunk_size=1280,
                     feature_init=None, streams=None, sr=None):
        """The detections of ``predict_clips(clips, padding, feature_init, chunk_size, streams, sr, patience, threshold,
        debounce_time)``: a list of (clip index, label, call index, score) for every call whose prediction is >= the
        threshold of its model, ordered by clip, then label (``labels()`` order), then call.  threshold: {model name:
        float} as in the reference (a model without one never fires), or one float for every model.  The scores stay
        on the device; only the event count and the events come back."""
        if not self.labels():
            raise ValueError("detect_clips needs at least one model")
        table = self._clip_table(patience, threshold, debounce_time)
        pcm, offsets = _concat_clips(clips)
        pcm, offsets, padding, check = self._clips_16k(pcm, offsets, padding, sr)
        raw, row_off, verified, dev = self._clip_call(pcm, offsets, padding, chunk_size, feature_init, streams, check)[:4]
        torch = _torch()
        labels = self.labels()
        ctx, stream = self.preprocessor.ctx, torch.cuda.current_stream(dev).cuda_stream
        n_ev = torch.zeros(1, dtype=torch.int32, device=dev)
        cap = min(int(row_off[-1]) * len(labels), 1 << 16)
        while True:                     # stateless: a call that found more events than the buffer holds runs again
            ev = torch.empty((max(cap, 1), 4), dtype=torch.int32, device=dev)
            ctx.detect_clips(table, max(float(debounce_time), 0.0), raw, verified, self.custom_verifier_threshold,
                             row_off, chunk_size, None, ev, cap, n_ev, stream)
            n = int(n_ev.item())
            if n <= cap:
                break
            cap = n
        e = ev[:n].cpu().numpy().view(_native.EVENT_DTYPE).reshape(-1)
        return list(zip(e["stream"].tolist(), [labels[j] for j in e["label"].tolist()], e["index"].tolist(),
                        e["score"].tolist()))

    def _clip_table(self, patience, threshold, debounce_time):
        """the label table of oww_detect_clips for predict's arguments, refused as predict refuses them"""
        if (patience != {} or debounce_time > 0) and threshold == {}:
            raise ValueError("Error! When using the `patience` argument, threshold "
                             "values must be provided via the `threshold` argument!")
        return self._detector_table(threshold, patience, debounce_time)

    def _clips_16k(self, pcm, offsets, padding, sr):
        """-> (pcm, offsets, padding, check_ingest) of the clips at 16 kHz: clips at other rates are resampled with their
        padding in one device launch"""
        offsets = np.ascontiguousarray(offsets, np.int64)
        rates = self._clip_rates(sr, offsets.size - 1, "the bulk clip path (predict_clips_ragged, bulk_predict)")
        if rates is None:
            return pcm, offsets, padding, sr is None
        d, off16 = self.preprocessor.resample_clips(pcm, offsets, rates, 16000 * int(padding))
        return d, off16, 0, False

    def _predict_ragged(self, pcm, offsets, padding, chunk_size, feature_init, want_features=False, streams=None,
                        check_ingest=True, table=None, debounce_time=0.0):
        """-> (scores, row_offsets, labels, embeddings [steps, 96] or None, step_offsets [N+1], feature_init rows).
        One oww_predict_clips_ragged call, then oww_detect_clips fills the rows of calls that stepped no chunk as
        Model.predict does (the previous prediction of single-output heads, zeros for multi-class heads, re-verified),
        zeroes each clip's first 5 calls (model.py:330-333) and applies `table` (_clip_table; None: no thresholds) and
        debounce_time.  check_ingest=False: the caller gave the clips' rate, so a device-ingest Model takes them too."""
        labels = self.labels()
        if table is None:
            table = self._clip_table({}, {}, 0.0)
        raw, row_off, verified, dev, emb, step_off, fi = self._clip_call(pcm, offsets, padding, chunk_size, feature_init,
                                                                         streams, check_ingest, want_features)
        out = self._clip_final(raw, row_off, chunk_size, table, debounce_time, verified, dev)
        emb = emb.cpu().numpy() if emb is not None else None
        return out, row_off, labels, emb, step_off, fi

    def _clip_final(self, raw, row_off, chunk_size, table, debounce_time, verified, dev):
        """oww_detect_clips over the raw rows -> host float32 [rows, n_labels]"""
        torch = _torch()
        rows = int(row_off[-1])
        if not table or not rows:
            return np.zeros((rows, len(table)), np.float32)
        final = torch.empty((rows, len(table)), dtype=torch.float32, device=dev)
        self.preprocessor.ctx.detect_clips(table, max(float(debounce_time), 0.0), raw, verified,
                                           self.custom_verifier_threshold, row_off, chunk_size, final, None, 0, None,
                                           torch.cuda.current_stream(dev).cuda_stream)
        return final.cpu().numpy()

    def _clip_call(self, pcm, offsets, padding, chunk_size, feature_init, streams, check_ingest, want_features=False):
        """One oww_predict_clips_ragged / _streams call -> (device raw rows, row_offsets [N+1], device p rows of the
        repeated calls' verifiers or None, device, device embeddings or None, step_offsets [N+1], feature_init rows)."""
        if check_ingest:
            self._no_ingest("the bulk clip path (predict_clips_ragged, bulk_predict)")
        if self._host_verifiers:
            warnings.warn(f"custom verifiers of {sorted(self._host_verifiers)} are not device-runnable (only the linear "
                          "pipeline of train_verifier_model is): predict_clips returns their models' unverified scores",
                          stacklevel=3)
        torch = _torch()
        chunk_size = int(chunk_size)
        limit = self.preprocessor.max_chunks * CHUNK
        if not 1 <= chunk_size <= limit:
            raise ValueError(f"chunk_size={chunk_size}: the bulk path takes 1 .. max_chunks*1280 = {limit} samples per call "
                             f"(max_chunks={self.preprocessor.max_chunks}); construct the Model with a larger max_chunks")
        offsets = np.ascontiguousarray(offsets, np.int64)
        n = offsets.size - 1
        if streams is not None:
            streams = np.asarray(streams, np.int64).ravel()
            if streams.size != n:
                raise ValueError(f"{streams.size} stream ids for {n} clips")
            if streams.size and (streams.min() < 0 or streams.max() >= self.n_streams):
                raise ValueError(f"stream ids must lie in [0, {self.n_streams})")
            self.preprocessor._ensure_streams()
        pad = 16000 * int(padding)
        lengths = np.diff(offsets)
        calls = np.array([_native.clip_schedule(chunk_size, int(x) + 2 * pad).size for x in lengths], np.int64)
        row_off = np.concatenate([[0], np.cumsum(calls)]).astype(np.int64)
        steps = calls * chunk_size // CHUNK                          # chunks stepped by a clip's calls (oww_clip_schedule)
        step_off = np.concatenate([[0], np.cumsum(steps)]).astype(np.int64)
        rows = int(row_off[-1])
        fi = feature_init if feature_init is not None else self.preprocessor._feature_init
        if fi is None:
            fi = self.preprocessor._get_embeddings(np.random.randint(-1000, 1000, 16000 * 4).astype(np.int16))
        fi = np.ascontiguousarray(fi, np.float32)
        dev = torch.device("cuda", self.preprocessor.device_index)
        if isinstance(pcm, torch.Tensor):
            d = pcm.to(device=dev, dtype=torch.int16, non_blocking=True).contiguous()
        else:
            d = torch.from_numpy(np.ascontiguousarray(pcm, np.int16)).to(dev)
        raw = torch.zeros((rows, max(self._n_cols, 1)), dtype=torch.float32, device=dev)
        need_emb = want_features or (chunk_size < CHUNK and bool(self._vbanks or self._svbanks))
        emb = torch.zeros((int(step_off[-1]), 96), dtype=torch.float32, device=dev) if need_emb else None
        stream = torch.cuda.current_stream(dev).cuda_stream
        self.preprocessor.ctx.predict_clips_ragged(d, offsets, pad, chunk_size, fi, raw, None, emb, stream,
                                                   clip_streams=streams)
        verified = self._verified_rows(calls, chunk_size, step_off, emb, fi, streams, dev) \
            if rows and chunk_size < CHUNK and (self._vbanks or self._svbanks) else None
        return raw, row_off, verified, dev, emb, step_off, fi

    def _verified_rows(self, calls, chunk_size, step_off, emb, fi, streams, dev):
        """_reverify on the rows of calls that step no chunk, on the device: -> float32 [rows, n_labels] (NaN where a
        label's model has no device verifier on the clip's stream, or the call steps) of the verifier's p on the clip's
        newest window ([feature_init rows | the clip's embeddings] up to its last step).  A row takes the slots of its
        clip's stream (streams[clip], or stream 0).  Calls with the same window share one verifier row; oww_detect_clips
        applies p to the predictions >= custom_verifier_threshold."""
        torch = _torch()
        labels = self.labels()
        n = calls.size
        rows = int(calls.sum())
        clip = np.repeat(np.arange(n), calls)
        local = np.arange(rows) - np.repeat(np.concatenate([[0], np.cumsum(calls)[:-1]]), calls)
        done = (local + 1) * chunk_size // CHUNK                     # chunks stepped up to and including the call
        rep = done == local * chunk_size // CHUNK
        row_stream = np.zeros(rows, np.int64) if streams is None else streams[clip]
        # [zero row | feature_init | every clip's embeddings]: a window's rows are gathered from it on the device
        table = torch.cat([torch.zeros((1, 96), dtype=torch.float32, device=dev), torch.from_numpy(fi).to(dev), emb])
        F = fi.shape[0]
        out = torch.full((rows, len(labels)), float("nan"), dtype=torch.float32, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        for mdl, st in list(self._vbanks.items()) + list(self._svbanks.items()):
            slots = np.where(self._has_model(mdl, row_stream), st["slots"][row_stream], -1)
            js = torch.tensor([j for j, lab in enumerate(labels) if self.get_parent_model_from_label(lab) == mdl],
                              dtype=torch.int64, device=dev)
            n_in = self.model_inputs[mdl]
            hit = rep & (slots >= 0)
            for slot in np.unique(slots[hit]):
                hit_rows = np.nonzero(hit & (slots == slot))[0]
                key = step_off[clip[hit_rows]] + clip[hit_rows] + done[hit_rows]    # one per (clip, window)
                _, first, inv = np.unique(key, return_index=True, return_inverse=True)
                r = hit_rows[first]
                q = F + done[r][:, None] - n_in + np.arange(n_in)[None, :]          # row of [fi | clip's embeddings]
                src = np.where(q < 0, 0, np.where(q < F, 1 + q, 1 + F + step_off[clip[r]][:, None] + q - F))
                p = torch.empty(r.size, dtype=torch.float32, device=dev)
                for a in range(0, r.size, 1 << 16):
                    b = min(r.size, a + (1 << 16))
                    feats = table[torch.from_numpy(src[a:b]).to(dev)].contiguous()
                    self.preprocessor.ctx.verifier_predict(st["bank"], int(slot), feats, b - a, p[a:b], stream)
                rt = torch.from_numpy(hit_rows).to(dev)
                out[rt[:, None], js[None, :]] = p[torch.from_numpy(inv.ravel()).to(dev)][:, None].expand(-1, js.numel())
        return out

    def _positive_frames_bulk(self, pcms, threshold=0.5, return_type="features", sr=None):
        """_get_positive_prediction_frames over many clips in one device call (padding 0, 1280-sample calls): per clip
        {label: stacked array} of what produced a score >= threshold.  sr: as in predict_clips_ragged; the audio context
        of clips at other rates is cut from their 16 kHz samples."""
        if return_type not in ("features", "audio"):
            raise ValueError("return_type must be 'features' or 'audio'")
        rates = self._clip_rates(sr, len(pcms), "_get_positive_prediction_frames")
        pcm, offsets = _concat_clips(pcms)
        if rates is not None:
            pcm, offsets = self.preprocessor.resample_clips(pcm, offsets, rates, 0)
            if return_type == "audio":
                host = pcm.cpu().numpy()
                pcms = [host[offsets[c]:offsets[c + 1]] for c in range(offsets.size - 1)]
        scores, row_off, labels, emb, step_off, fi = self._predict_ragged(pcm, offsets, 0, CHUNK, None,
                                                                          want_features=return_type == "features",
                                                                          check_ingest=sr is None)
        n_in = {lab: self.model_inputs[self.get_parent_model_from_label(lab)] for lab in labels}
        res = []
        for c, data in enumerate(pcms):
            hits = {}
            for s in range(int(row_off[c + 1] - row_off[c])):
                for j, lab in enumerate(labels):
                    if scores[row_off[c] + s, j] < threshold:
                        continue
                    if return_type == "features":
                        hits.setdefault(lab, []).append(_window(fi, emb, step_off[c], s + 1, n_in[lab])[None])
                    else:
                        i = s * CHUNK
                        context = data[max(0, i - 16000 * 3):i + 16000]
                        if len(context) == 16000 * 4:
                            hits.setdefault(lab, []).append(context)
            res.append({lab: np.vstack(v) for lab, v in hits.items() if v})
        return res

    def labels(self):
        """Output labels in score-column order (binary heads: model name; multi-class: mapped labels)."""
        labs = []
        for mdl in self.models:
            if self.model_outputs[mdl] == 1:
                labs.append(mdl)
            else:
                labs += list(self.class_mapping[mdl].values())
        return labs

    def predict_clips_array(self, clips, padding=1, feature_init=None, patience={}, threshold={}, debounce_time=0.0):
        """-> (float32 [N, steps, n_labels], labels) with the first-5-steps zeroing of model.py:330-333 applied, and
        patience, threshold and debounce_time as in ``predict`` (oww_detect_clips on the device).  Device verifiers
        apply (stream 0's); host-only verifiers do not, and a warning says so."""
        self._no_ingest("predict_clips_array")
        table = self._clip_table(patience, threshold, debounce_time)
        if self._host_verifiers:
            warnings.warn(f"custom verifiers of {sorted(self._host_verifiers)} are not device-runnable (only the linear "
                          "pipeline of train_verifier_model is): predict_clips returns their models' unverified scores",
                          stacklevel=2)
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
        dev = torch.device("cuda", self.preprocessor.device_index)
        d = clips.to(dev, non_blocking=True) if isinstance(clips, torch.Tensor) else torch.from_numpy(clips).to(dev)
        raw = torch.zeros((N, steps, max(self._n_cols, 1)), dtype=torch.float32, device=dev)
        self.preprocessor.ctx.predict_clips(d, N, S, 16000 * padding, fi, raw, torch.cuda.current_stream(d.device).cuda_stream)
        row_off = np.arange(N + 1, dtype=np.int64) * steps
        out = self._clip_final(raw, row_off, CHUNK, table, debounce_time, None, dev)
        return out.reshape(N, steps, len(table)), self.labels()


class StreamState:
    """Streams exported by ``Model.export_streams``, in export order: ``records`` (torch.uint8 [n, record bytes], the
    device state of include/owwb200.h), ``key`` (the configuration the records are valid under), ``labels``, and per
    stream what the host keeps: ``pending`` (int16 samples not yet stepped), ``history`` / ``counts`` ({label: float32
    [30, n] prediction ring, int64 [n] predictions appended}), ``audio`` (None without an audio history, else the
    history: int16 [n, H] oldest first, int64 [n] sample positions, bool [n] whether the samples held not yet stepped
    count in ``raw_data_buffer``), ``ingest`` (None without device ingest, else the resampler state: int32 [n] rates, int64
    [n] input samples since each resampler's restart, int32 [n] staged counts, int16 [n, max staged] staged 16 kHz samples,
    int16 [n, 128] filter histories), ``detection`` (None, or per stream None or the (threshold, patience, debounce_time)
    of ``Model.set_stream_detection``).  ``to(device)`` moves the records; on the CPU it pickles."""

    def __init__(self, records, key, labels, pending, history, counts, audio=None, ingest=None, detection=None):
        self.records, self.key, self.labels = records, int(key), list(labels)
        self.pending, self.history, self.counts = pending, history, counts
        self.audio = audio
        self.ingest = ingest
        self.detection = detection

    def __len__(self):
        return len(self.pending)

    def to(self, device):
        return StreamState(self.records.to(device), self.key, self.labels, self.pending, self.history, self.counts,
                           self.audio, self.ingest, self.detection)


def _concat_clips(clips):
    """[N,S] array / tensor or a sequence of 1-D int16 arrays -> (one int16 array or tensor, int64 offsets [N+1])"""
    torch = _torch()
    if isinstance(clips, torch.Tensor) and clips.dim() == 2:
        n, s = clips.shape
        return clips.reshape(-1), np.arange(n + 1, dtype=np.int64) * s
    if isinstance(clips, np.ndarray) and clips.ndim == 2:
        n, s = clips.shape
        return np.ascontiguousarray(clips, np.int16).reshape(-1), np.arange(n + 1, dtype=np.int64) * s
    parts = [np.asarray(c).astype(np.int16, copy=False).ravel() for c in clips]
    offsets = np.concatenate([[0], np.cumsum([p.size for p in parts])]).astype(np.int64)
    pcm = np.concatenate(parts) if parts else np.zeros(0, np.int16)
    return pcm, offsets


def _rows_to_dicts(scores, row_off, labels):
    return [[{lab: float(v) for lab, v in zip(labels, row)} for row in scores[row_off[c]:row_off[c + 1]]]
            for c in range(row_off.size - 1)]


def _window(fi, emb, step0, done, n_in):
    """the newest n_in feature rows of a clip after `done` of its steps: rows of [feature_init | its embeddings] ending
    at row len(fi) + done, rows before the first read as zeros (AudioFeatures.get_features) -> [n_in, 96]"""
    rows = np.concatenate([fi, emb[step0:step0 + done]]) if done else fi
    w = np.zeros((n_in, 96), np.float32)
    k = min(n_in, rows.shape[0])
    if k:
        w[n_in - k:] = rows[rows.shape[0] - k:]
    return w
