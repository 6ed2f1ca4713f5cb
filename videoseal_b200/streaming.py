"""RGB24 clip I/O around embed/detect: the two inner functions of the reference's streaming CLI, same names and arguments
(inference_streaming.py:23-33 `embed_video_clip`, :116-124 `detect_video_clip`), running through `vsb_frames_host_u8`.

The reference converts uint8 HWC -> float32 CHW on the host, calls the model, and converts back; here the uint8 frames cross
PCIe as they are (4x fewer bytes each way) and both conversions run on the GPU inside the chunked, copy/compute-overlapped
host entry point.  Results are those of the reference's arithmetic: x = u8 / 255, u8 = (imgs_w * 255).byte().
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from .model import _DEF_INTERP, Videoseal


def _as_u8_clip(clip) -> np.ndarray:
    a = clip.numpy() if isinstance(clip, torch.Tensor) else np.asarray(clip)
    if a.dtype != np.uint8 or a.ndim != 4 or a.shape[3] != 3:
        raise ValueError("clip must be uint8 [F, H, W, 3] (RGB24 frames)")
    return np.ascontiguousarray(a)


def _run(model: Videoseal, clip: np.ndarray, msgs, want_frames: bool, want_logits: bool, lowres_attenuation: bool, is_video: bool):
    F_, H, W = clip.shape[0], clip.shape[1], clip.shape[2]
    if want_logits and model.pixelwise:
        raise NotImplementedError("streaming detection returns one logit vector per frame; a pixel-wise model's maps come from "
                                  "model.detect()")
    nbits = model.spec["nbits"]
    out = np.empty_like(clip) if want_frames else None
    logits = np.empty((F_, 1 + nbits), dtype=np.float32) if want_logits else None
    m8 = None
    n_msgs = 0
    if want_frames:
        if msgs is None:
            msgs = model.get_random_msg(1 if is_video else F_)
        m8 = (msgs.detach().cpu() > 0.5).to(torch.uint8).contiguous().numpy()
        if m8.ndim != 2 or m8.shape[1] != nbits or m8.shape[0] not in (1, F_) or (is_video and m8.shape[0] != 1):
            raise ValueError("msgs must be [1, nbits] for a video clip (or [F, nbits] with is_video=False)")
        n_msgs = m8.shape[0]
    interp = _DEF_INTERP
    flags = model._flags(interp, lowres_attenuation)
    _lib.check(_lib.lib().vsb_frames_host_u8(
        model._handle(), clip.ctypes.data_as(C.c_void_p), m8.ctypes.data_as(C.c_void_p) if m8 is not None else None, n_msgs,
        out.ctypes.data_as(C.c_void_p) if out is not None else None,
        logits.ctypes.data_as(C.c_void_p) if logits is not None else None,
        F_, H, W, model.step_size if is_video else 1, _lib.VIDEO_MODES[model.video_mode], model._chunk_keys(is_video, F_),
        float(model.blender.scaling_i), float(model.blender.scaling_w), flags))
    return out, (torch.from_numpy(logits) if logits is not None else None), msgs


def embed_video_clip(model: Videoseal, clip: np.ndarray, msgs: torch.Tensor) -> np.ndarray:
    """inference_streaming.py:23-33: uint8 [F,H,W,3] -> watermarked uint8 [F,H,W,3] (is_video=True, lowres_attenuation=True)."""
    out, _, _ = _run(model, _as_u8_clip(clip), msgs, True, False, True, True)
    return out


def detect_video_clip(model: Videoseal, clip: np.ndarray) -> torch.Tensor:
    """inference_streaming.py:116-124: uint8 [F,H,W,3] -> logits of the message bits [F, nbits] (column 0 dropped)."""
    _, logits, _ = _run(model, _as_u8_clip(clip), None, False, True, False, True)
    return logits[:, 1:]


def embed_detect_video_clip(model: Videoseal, clip: np.ndarray, msgs: torch.Tensor = None, lowres_attenuation: bool = True,
                            is_video: bool = True):
    """embed_video_clip followed by detect_video_clip on the watermarked uint8 frames, in one pass over the GPU.
    Returns (frames_w uint8 [F,H,W,3], preds [F, 1+nbits], msgs)."""
    return _run(model, _as_u8_clip(clip), msgs, True, True, lowres_attenuation, is_video)


# ---------------------------------------------------------------------------------------------------------------------
# The outer loops of the reference's streaming CLI (inference_streaming.py:35-114 `embed_video`, :126-164 `detect_video`,
# :167-200 main): rawvideo RGB24 frames from a decoder pipe, fixed-size chunks through the clip functions above, frames to an
# encoder pipe.  The reference reads, computes and writes strictly in turn; here a reader thread and a writer thread keep the
# pipes busy while the GPU works on the chunk in between (bounded queues = a small host ring), which is what decides the
# frames/s of a real transcode once the model itself runs at thousands of frames per second.
import queue
import shutil
import subprocess
import threading


def iter_rawvideo_chunks(stream, width: int, height: int, chunk_size: int):
    """uint8 [n, H, W, 3] chunks (n == chunk_size except for the last one) from a binary stream of RGB24 frames"""
    frame_bytes = width * height * 3
    want = frame_bytes * chunk_size
    while True:
        buf = stream.read(want)
        if not buf:
            return
        while len(buf) < want:                      # unbuffered pipes may return short reads: only EOF ends a chunk early
            more = stream.read(want - len(buf))
            if not more:
                break
            buf += more
        n = len(buf) // frame_bytes
        if n == 0:
            return
        yield np.frombuffer(buf[: n * frame_bytes], np.uint8).reshape(n, height, width, 3)
        if n < chunk_size:
            return


def _put(q: "queue.Queue", item, alive) -> bool:
    """q.put that gives up when `alive()` turns false (the other side of the queue has died or left): a plain blocking put on
    a full queue would wait forever for a consumer that no longer exists"""
    while alive():
        try:
            q.put(item, timeout=0.1)
            return True
        except queue.Full:
            continue
    return False


def _prefetched(it, depth: int):
    """run iterator `it` in a thread, `depth` items ahead; the producer stops when the consumer goes away (generator closed or
    garbage-collected, e.g. after an exception in the consumer's loop body)"""
    q: "queue.Queue" = queue.Queue(maxsize=max(1, depth))
    end = object()
    stop = threading.Event()

    def work():
        try:
            for x in it:
                if not _put(q, x, lambda: not stop.is_set()):
                    return
            _put(q, end, lambda: not stop.is_set())
        except BaseException as e:   # surfaced in the consumer
            _put(q, e, lambda: not stop.is_set())

    threading.Thread(target=work, daemon=True).start()
    try:
        while True:
            x = q.get()
            if x is end:
                return
            if isinstance(x, BaseException):
                raise x
            yield x
    finally:
        stop.set()


def embed_stream(model, src, dst, width: int, height: int, chunk_size: int, msgs: torch.Tensor = None, prefetch: int = 2,
                 clip_fn=None) -> torch.Tensor:
    """Watermark every frame of the RGB24 stream `src` into `dst` (file-like objects) with ONE message; returns the message.
    Same chunking as inference_streaming.py:83-107 (full chunks, then the partial tail)."""
    clip_fn = clip_fn or embed_video_clip
    if msgs is None:
        msgs = model.get_random_msg()
    out_q: "queue.Queue" = queue.Queue(maxsize=max(1, prefetch))
    err = []

    def writer():
        try:
            while True:
                a = out_q.get()
                if a is None:
                    return
                dst.write(a.tobytes())
        except BaseException as e:
            err.append(e)

    wt = threading.Thread(target=writer, daemon=True)
    wt.start()
    chunks = _prefetched(iter_rawvideo_chunks(src, width, height, chunk_size), prefetch)
    try:
        for chunk in chunks:
            # a GPU faster than the encoder keeps out_q full: the put must notice a writer that died (BrokenPipe from ffmpeg)
            if err or not _put(out_q, clip_fn(model, chunk, msgs), lambda: wt.is_alive() and not err):
                break
    finally:
        chunks.close()                                   # stops the reader thread
        _put(out_q, None, lambda: wt.is_alive())         # sentinel, unless the writer is already gone
        wt.join()
    if err:
        raise err[0]
    return msgs


def detect_stream(model, src, width: int, height: int, chunk_size: int, include_tail: bool = False, prefetch: int = 2,
                  clip_fn=None) -> torch.Tensor:
    """Soft message (mean of the per-frame bit logits) of an RGB24 stream.  The reference only feeds FULL chunks to the
    detector (inference_streaming.py:155-156: frames after the last multiple of chunk_size are never looked at);
    include_tail=True also uses the partial last chunk."""
    clip_fn = clip_fn or detect_video_clip
    soft = []
    for chunk in _prefetched(iter_rawvideo_chunks(src, width, height, chunk_size), prefetch):
        if len(chunk) == chunk_size or include_tail:
            soft.append(clip_fn(model, chunk))
    if not soft:
        raise ValueError("no full chunk in the stream: lower chunk_size or pass include_tail=True")
    return torch.cat(soft, dim=0).mean(dim=0)


def _probe(path: str):
    if shutil.which("ffprobe") is None or shutil.which("ffmpeg") is None:
        raise RuntimeError("ffmpeg / ffprobe not found on PATH: use embed_stream / detect_stream on rawvideo RGB24 streams instead")
    import json
    info = json.loads(subprocess.check_output(["ffprobe", "-v", "error", "-select_streams", "v:0", "-show_entries",
                                               "stream=width,height,r_frame_rate", "-of", "json", path]))["streams"][0]
    num, den = info["r_frame_rate"].split("/")
    return int(info["width"]), int(info["height"]), float(num) / float(den)


def embed_video(model, input_path: str, output_path: str, chunk_size: int, crf: int = 23) -> torch.Tensor:
    """inference_streaming.py:35-114: decode with ffmpeg -> embed -> encode (libx264, yuv420p); writes the message next to the video"""
    w, h, fps = _probe(input_path)
    dec = subprocess.Popen(["ffmpeg", "-v", "error", "-i", input_path, "-f", "rawvideo", "-pix_fmt", "rgb24", "-s", f"{w}x{h}",
                            "-r", str(fps), "pipe:"], stdout=subprocess.PIPE)
    enc = subprocess.Popen(["ffmpeg", "-v", "error", "-y", "-f", "rawvideo", "-pix_fmt", "rgb24", "-s", f"{w}x{h}", "-r", str(fps),
                            "-i", "pipe:", "-vcodec", "libx264", "-pix_fmt", "yuv420p", "-crf", str(crf), "-r", str(fps), output_path],
                           stdin=subprocess.PIPE)
    try:
        msgs = embed_stream(model, dec.stdout, enc.stdin, w, h, chunk_size)
    finally:
        dec.stdout.close()
        enc.stdin.close()
        dec.wait()
        enc.wait()
    with open(output_path.rsplit(".", 1)[0] + ".txt", "w") as f:
        f.write("".join(str(int(b)) for b in msgs[0]))
    return msgs


def detect_video(model, input_path: str, chunk_size: int) -> torch.Tensor:
    """inference_streaming.py:126-164"""
    w, h, _ = _probe(input_path)
    dec = subprocess.Popen(["ffmpeg", "-v", "error", "-i", input_path, "-f", "rawvideo", "-pix_fmt", "rgb24", "pipe:"], stdout=subprocess.PIPE)
    try:
        return detect_stream(model, dec.stdout, w, h, chunk_size)
    finally:
        dec.stdout.close()
        dec.wait()


def main(argv=None):
    """python -m videoseal_b200.streaming --input in.mp4 --output_dir outputs  (inference_streaming.py:167-200)"""
    import argparse
    import os
    ap = argparse.ArgumentParser(description="streaming video watermarking on the H100 (CUDA) backend")
    ap.add_argument("--input", required=True)
    ap.add_argument("--output_dir", default="outputs")
    ap.add_argument("--model", default="videoseal")
    ap.add_argument("--chunk_size", type=int, default=64)
    ap.add_argument("--crf", type=int, default=23)
    a = ap.parse_args(argv)
    from . import load
    model = load(a.model).eval().to("cuda")
    os.makedirs(a.output_dir, exist_ok=True)
    out = os.path.join(a.output_dir, os.path.basename(a.input))
    msgs = embed_video(model, a.input, out, a.chunk_size, a.crf)
    soft = detect_video(model, out, a.chunk_size)
    acc = ((soft > 0) == (msgs[0].to(soft.device) > 0.5)).float().mean().item()
    print(f"Saved watermarked video to {out}; binary message accuracy after re-encoding: {acc * 100:.2f}%")


if __name__ == "__main__":
    main()
