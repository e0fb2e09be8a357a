"""Service layer over the batched driver (SURVEY.md section 8f, row N2): the HTTP endpoint of
``tools/diffusion/flask_api.py:24-60`` and the framed TCP loop of ``tools/diffusion/tcp_api.py:24-75``, on the standard
library (flask / flask_cors / soundfile / librosa are not in this image, and the feature / pitch extractors the reference
calls through ``SVCInference`` are out of scope, SURVEY.md section 2).

What carries over from the reference:
  * ``POST /voiceChangeModel`` with the multipart / form fields ``sample`` (a wav file), ``fPitchChange``, ``sSpeakId``,
    ``sampleRate``; the response is a wav attachment at the caller's sample rate (flask_api.py:24-60);
  * the TCP protocol: fixed frames of ``3 * 44100`` float32 samples in, the same number of float32 samples out, silence
    answered with zeros without running the model (tcp_api.py:40-75).
What is new: requests do not each run a B=1 model call.  A request is turned into (features [T,E], f0 [T]) segments by the
``frontend`` callable the deployer supplies (the reference's extractors: ``SVCInference`` slicing + ContentVec + pitch),
and concurrent requests are merged into ONE BatchedSynthesizer call per collection window -- the reference serves
``threaded=True`` over a single shared model (flask_api.py:86), which on this path would serialise on the module's work
buffers; here a single worker thread owns the model and the handler threads only queue work.

``frontend(audio float32 [n], sr, pitch_adjust, speaker_id) -> list of (features [T,E] CUDA, f0 [T] CUDA, n_samples)``
``resample(audio, sr_in, sr_out) -> audio`` (identity when the rates match; the reference uses librosa.resample):
pass ``device_resampler()``, the package's own Kaiser-sinc kernel.  The same kernel is the first stage of a ``frontend``
whose content encoder wants 16 kHz audio (modules/feature_extractors/base.py:25)::

    from fish_diffusion_b200 import resample
    def frontend(audio, sr, pitch_adjust, speaker_id):
        wav = torch.from_numpy(audio).cuda()[None]             # [1, n] at the model rate
        wav16 = resample(wav, sr, 16000)                       # 44.1 k -> 16 k for HuBERT / ContentVec, on the device
        ...
    srv = make_http_server(worker, frontend, model_sr=44100, resample=device_resampler())
"""
from __future__ import annotations

import io
import queue
import threading
import wave
from http.server import BaseHTTPRequestHandler, ThreadingHTTPServer
from typing import Callable, List, Optional

import numpy as np


def wav_bytes(audio: np.ndarray, sr: int) -> bytes:
    """float32 mono -> 16-bit PCM wav (what soundfile.write(..., format="wav") returns for the VST client)."""
    pcm = (np.clip(np.asarray(audio, dtype=np.float32), -1.0, 1.0) * 32767.0).astype("<i2")
    buf = io.BytesIO()
    with wave.open(buf, "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(int(sr))
        w.writeframes(pcm.tobytes())
    return buf.getvalue()


def read_wav(data: bytes):
    """16-bit / 32-bit-float PCM wav -> (float32 mono, sample rate)."""
    with wave.open(io.BytesIO(data), "rb") as w:
        sr, n, ch, sw = w.getframerate(), w.getnframes(), w.getnchannels(), w.getsampwidth()
        raw = w.readframes(n)
    if sw == 2:
        a = np.frombuffer(raw, dtype="<i2").astype(np.float32) / 32768.0
    elif sw == 4:
        a = np.frombuffer(raw, dtype="<f4").astype(np.float32)
    else:
        raise ValueError(f"unsupported sample width {sw}")
    if ch > 1:
        a = a.reshape(-1, ch).mean(axis=1)
    return a, sr


class BatchingWorker:
    """One thread owns the synthesizer; requests queue their segments and wait for their waveform.  All segments that
    arrive within `window_s` of the first one are synthesised in ONE BatchedSynthesizer call."""

    def __init__(self, synthesizer: Callable[[List, List], List], window_s: float = 0.01, max_segments: int = 64):
        self.synth, self.window_s, self.max_segments = synthesizer, window_s, max_segments
        self.q: "queue.Queue" = queue.Queue()
        self.batches = 0
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()

    def submit(self, segments):
        """segments: list of (features, f0); blocks until their waveforms are ready and returns them in order."""
        done = threading.Event()
        slot = {"segments": segments, "done": done, "out": None, "err": None}
        self.q.put(slot)
        done.wait()
        if slot["err"] is not None:
            raise slot["err"]
        return slot["out"]

    def close(self):
        self.q.put(None)
        self._t.join(timeout=5)

    def _run(self):
        while True:
            slot = self.q.get()
            if slot is None:
                return
            slots, n = [slot], len(slot["segments"])
            try:
                while n < self.max_segments:
                    nxt = self.q.get(timeout=self.window_s)
                    if nxt is None:
                        self.q.put(None)
                        break
                    slots.append(nxt)
                    n += len(nxt["segments"])
            except queue.Empty:
                pass
            feats = [f for s in slots for f, _ in s["segments"]]
            f0s = [p for s in slots for _, p in s["segments"]]
            try:
                wavs = self.synth(feats, f0s) if feats else []
                self.batches += 1
                i = 0
                for s in slots:
                    k = len(s["segments"])
                    s["out"] = wavs[i:i + k]
                    i += k
            except Exception as ex:  # noqa: BLE001 -- every waiting request gets the error
                for s in slots:
                    s["err"] = ex
            for s in slots:
                s["done"].set()


def _to_numpy(w):
    return w.detach().float().cpu().numpy() if hasattr(w, "detach") else np.asarray(w, dtype=np.float32)


def convert(worker: BatchingWorker, frontend, audio, sr, pitch_adjust, speaker_id, model_sr=44100):
    """audio -> segments (frontend) -> one batched synthesis -> concatenated waveform (the role of SVCInference.forward,
    tools/diffusion/inference.py:85-162, whose per-segment B=1 loop this replaces)."""
    segs = frontend(np.asarray(audio, dtype=np.float32), sr, pitch_adjust, speaker_id)
    if not segs:
        return np.zeros(0, dtype=np.float32)
    wavs = worker.submit([(f, p) for f, p, _ in segs])
    return np.concatenate([_to_numpy(w)[:n] for w, (_, _, n) in zip(wavs, segs)])


def _parse_multipart(body: bytes, content_type: str):
    """Minimal multipart/form-data parser (fields + one file), enough for the VST client's request."""
    fields, files = {}, {}
    if "boundary=" not in content_type:
        return fields, files
    boundary = ("--" + content_type.split("boundary=", 1)[1].strip().strip('"')).encode()
    for part in body.split(boundary):
        part = part.strip(b"\r\n")
        if not part or part == b"--" or b"\r\n\r\n" not in part:
            continue
        head, data = part.split(b"\r\n\r\n", 1)
        head = head.decode("utf-8", "replace")
        name = head.split('name="', 1)[1].split('"', 1)[0] if 'name="' in head else None
        if name is None:
            continue
        if "filename=" in head:
            files[name] = data
        else:
            fields[name] = data.decode("utf-8", "replace")
    return fields, files


def device_resampler(device="cuda"):
    """The ``resample=`` callable of make_http_server on the package's resampling kernel: (audio float32 [n] numpy,
    sr_in, sr_out) -> float32 [ceil(n * sr_out / sr_in)] numpy.  Uploads, runs fd_resample_fwd, downloads; equal rates
    pass the array through.  Replaces librosa.load(..., sr=model_sr) / librosa.resample(..., target_sr=daw_sample) of
    flask_api.py:42,53."""
    import torch
    from .resample import resample

    def run(audio, sr_in, sr_out):
        audio = np.ascontiguousarray(audio, dtype=np.float32)
        if int(sr_in) == int(sr_out) or audio.size == 0:
            return audio
        return resample(torch.from_numpy(audio).to(device), sr_in, sr_out).cpu().numpy()

    return run


def make_http_server(worker: BatchingWorker, frontend, host="0.0.0.0", port=6842, model_sr=44100,
                     resample: Optional[Callable] = None, default_speaker: Optional[int] = None):
    """ThreadingHTTPServer with the reference's route (flask_api.py:24-60; port 6842 is what the VST plugin expects).
    `resample(audio, sr_in, sr_out)` converts the request to `model_sr` and the answer to the caller's `sampleRate`;
    pass ``device_resampler()``.  The default None passes audio through unchanged, which is right only when the
    caller's rate is the model's."""
    resample = resample or (lambda a, sr_in, sr_out: a)

    class Handler(BaseHTTPRequestHandler):
        def log_message(self, *a):  # quiet
            pass

        def do_POST(self):
            if self.path.rstrip("/") != "/voiceChangeModel":
                self.send_error(404)
                return
            body = self.rfile.read(int(self.headers.get("Content-Length", 0)))
            fields, files = _parse_multipart(body, self.headers.get("Content-Type", ""))
            if "sample" not in files:
                self.send_error(400, "multipart field 'sample' (wav file) missing")
                return
            try:
                pitch = float(fields.get("fPitchChange", 0))
                spk = int(fields.get("sSpeakId", 0)) if default_speaker is None else int(default_speaker)
                daw_sr = int(float(fields.get("sampleRate", 0))) or model_sr
                audio, sr = read_wav(files["sample"])
                audio = resample(audio, sr, model_sr)
                out = convert(worker, frontend, audio, model_sr, pitch, spk, model_sr)
                data = wav_bytes(resample(out, model_sr, daw_sr), daw_sr)
            except Exception as ex:  # noqa: BLE001
                self.send_error(500, repr(ex)[:200])
                return
            self.send_response(200)
            self.send_header("Content-Type", "audio/wav")
            self.send_header("Content-Disposition", 'attachment; filename="temp.wav"')
            self.send_header("Content-Length", str(len(data)))
            self.send_header("Access-Control-Allow-Origin", "*")          # flask_cors.CORS(app)
            self.end_headers()
            self.wfile.write(data)

    return ThreadingHTTPServer((host, port), Handler)


def tcp_frame_loop(conn, worker: BatchingWorker, frontend, frame_samples=3 * 44100, sr=44100, pitch_adjust=4, speaker_id=0,
                   silence_peak=1e-4, max_frames: Optional[int] = None):
    """tcp_api.py:40-75: read float32 frames of `frame_samples`, answer each with the converted frame (zeros for a silent
    frame, padded / cut to the frame length).  Returns the number of frames served when the peer closes."""
    frame_bytes, buff, served = 4 * frame_samples, b"", 0
    while max_frames is None or served < max_frames:
        data = conn.recv(frame_bytes)
        if not data:
            break
        buff += data
        while len(buff) >= frame_bytes:
            chunk, buff = buff[:frame_bytes], buff[frame_bytes:]
            audio = np.frombuffer(chunk, dtype=np.float32)
            peak = float(np.abs(audio).max()) if audio.size else 0.0
            if peak < silence_peak:          # a silent frame is answered without a model call (tcp_api.py:52-58 gates on
                                             # librosa.effects.split; librosa is absent here, the gate is a peak threshold)
                conn.sendall(np.zeros(frame_samples, dtype=np.float32).tobytes())
            else:
                out = convert(worker, frontend, audio, sr, pitch_adjust, speaker_id, sr)
                if len(out) < frame_samples:
                    out = np.pad(out, (0, frame_samples - len(out)))
                conn.sendall(np.asarray(out[:frame_samples], dtype=np.float32).tobytes())
            served += 1
    return served


def pack_frame(audio: np.ndarray) -> bytes:
    return np.asarray(audio, dtype=np.float32).tobytes()


def unpack_frame(data: bytes) -> np.ndarray:
    return np.frombuffer(data, dtype=np.float32)


__all__ = ["BatchingWorker", "convert", "device_resampler", "make_http_server", "tcp_frame_loop", "wav_bytes", "read_wav", "pack_frame",
           "unpack_frame"]
