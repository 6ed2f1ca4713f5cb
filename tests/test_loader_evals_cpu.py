"""Host-side logic that needs no GPU: raw-training-checkpoint loading (SURVEY 8(f)3, utils/cfg.py:50-85,156-178 of the
reference), the metrics of the evaluation slice (8(f)4, evals/metrics.py) and the speed tester's bookkeeping."""
import argparse
import math
import os

import pytest
import torch

from oracle import restate
from tests.util import load_card, tmpdir
import videoseal_b200
from videoseal_b200 import cfg as vcfg
from videoseal_b200.evals import metrics, speed


def _training_ckpt(card_name, emb_model, ext_model, as_namespace=False):
    card = load_card(card_name)
    spec = restate.spec_from_card(card)
    args = dict(card["args"])
    args.update({"embedder_config": "configs/embedder.yaml", "extractor_config": "configs/extractor.yaml",
                 "embedder_model": emb_model, "extractor_model": ext_model, "lr": 1e-4, "epochs": 3})
    path = tmpdir() / f"train_{card_name}_{int(as_namespace)}.pth"
    # a small stand-in state dict is enough: load_state_dict keeps what it is given, nothing is finalised without a GPU
    sd = {"embedder.unet.outc.bias": torch.zeros(spec["unet"]["out_channels"])}
    torch.save({"args": argparse.Namespace(**args) if as_namespace else args, "model": sd, "epoch": 3}, path)
    return path, card


@pytest.mark.parametrize("card_name,emb,ext", [("videoseal_1.0", "unet_small2_yuv_quant", "convnext_tiny"),
                                               ("pixelseal", "unet_base_yuv_quant", "convnext_tiny"),
                                               ("chunkyseal", "unet_sweep_3", "convnext_sweep_3_prop_stride2")])
def test_training_checkpoint_resolves_to_the_cards_architecture(built_lib, card_name, emb, ext):
    path, card = _training_ckpt(card_name, emb, ext)
    got = vcfg.spec_from_card(vcfg.get_config_from_checkpoint(path))
    want = vcfg.spec_from_card(card)
    assert got == want
    model = vcfg.setup_model_from_checkpoint(str(path))
    assert model.spec == want and "embedder.unet.outc.bias" in model.state_dict()


def test_training_checkpoint_args_as_namespace_and_card_name_passthrough(built_lib):
    path, card = _training_ckpt("videoseal_1.0", "unet_small2_yuv_quant", "convnext_tiny", as_namespace=True)
    assert vcfg.spec_from_card(vcfg.get_config_from_checkpoint(path)) == vcfg.spec_from_card(card)
    with pytest.raises(NotImplementedError):
        vcfg.setup_model_from_checkpoint("baseline/hidden")
    with pytest.raises(FileNotFoundError):
        vcfg.setup_model_from_checkpoint("no_such_card")
    from videoseal_b200.utils.cfg import setup_model_from_checkpoint as alias   # the reference's import path
    assert alias is vcfg.setup_model_from_checkpoint


def test_unknown_preset_is_rejected_at_load_time():
    path, _ = _training_ckpt("videoseal_1.0", "unet_small2_yuv_quant", "sam_small")
    with pytest.raises(NotImplementedError):
        vcfg.get_config_from_checkpoint(path)


def test_videoseal_0_0_card_is_rejected_by_the_product_loader():
    """configs[0] runs on the reference's CPU path only (oracle); the CUDA package has no ViT extractor and no CPU fallback"""
    with pytest.raises(NotImplementedError):
        vcfg.spec_from_card(load_card("videoseal_0.0"))


def test_metrics_match_the_oracle_and_closed_forms():
    g = torch.Generator().manual_seed(0)
    x = torch.rand(3, 3, 32, 40, generator=g)
    y = (x + 0.01 * torch.randn(3, 3, 32, 40, generator=g)).clamp(0, 1)
    assert torch.allclose(metrics.psnr(y, x), restate.psnr(y, x))
    assert metrics.psnr(y, x, is_video=True).ndim == 0
    mse = ((255 * (y - x)) ** 2).mean().item()
    assert metrics.psnr(y, x, is_video=True).item() == pytest.approx(20 * math.log10(255) - 10 * math.log10(mse), abs=1e-4)
    assert metrics.linf(y, x).item() == pytest.approx(255 * (y - x).abs().max().item())
    logits = torch.tensor([[9.0, 1.0, -1.0, 2.0, -3.0], [0.0, -1.0, -1.0, -2.0, 3.0]])
    msgs = torch.tensor([[1, 0, 1, 0], [1, 1, 0, 0]])
    acc = metrics.bit_accuracy(logits[:, 1:], msgs)
    assert acc.tolist() == [1.0, 0.25]
    assert torch.equal(acc, restate.bit_accuracy(logits, msgs))
    pv = metrics.pvalue(logits[:, 1:], msgs)
    assert pv[0].item() == pytest.approx(0.5 ** 4) and pv[1].item() == pytest.approx(1 - 0.5 ** 4)
    cap = metrics.capacity(logits[:, 1:], msgs)
    assert cap[0].item() == pytest.approx(4.0)
    assert cap[1].item() == pytest.approx(4 * (1 + 0.25 * math.log2(0.25) + 0.75 * math.log2(0.75)))
    pix = torch.zeros(1, 2, 4, 4)
    pix[0, 0] = 1.0
    pix[0, 1, :1] = 1.0    # 4 of 16 pixels vote 1 -> bit 0
    assert metrics.bit_accuracy(pix, torch.tensor([[1, 0]])).item() == 1.0


class _FakeModel:
    def __init__(self):
        self.calls = []

    def embed(self, imgs, msgs=None, is_video=True, interpolation=None, lowres_attenuation=False):
        self.calls.append(("embed", tuple(imgs.shape), is_video, lowres_attenuation))
        return {"imgs_w": imgs}

    def detect(self, imgs, is_video=True):
        self.calls.append(("detect", tuple(imgs.shape), is_video))
        return {"preds": torch.zeros(len(imgs), 5)}

    def extract_message(self, imgs, aggregation="avg", interpolation=None):
        self.calls.append(("extract", tuple(imgs.shape), aggregation))
        return torch.zeros(1, 4, dtype=torch.bool)


def test_speed_tester_bookkeeping_matches_the_reference_semantics():
    m = _FakeModel()
    items = list(speed.synthetic_items(2, True, 10, 16, 24, "cpu"))
    res = speed.SpeedTester("cpu").test_speed(m, items, is_video=True, num_frames=8, num_runs=2, warmup_runs=1)
    # per item: 1 warm-up (embed + extract) + 2 timed embeds + 2 timed extracts, all on the first 8 frames
    assert len(m.calls) == 2 * (2 + 2 + 2) and all(c[1][0] == 8 for c in m.calls)
    assert res["image_shape"] == ["10x16x24", "10x16x24"] and len(res["embedding_time"]) == 2
    assert res["avg_embedding_ms_per_frame"] == pytest.approx(res["avg_embedding_time"] / 8 * 1000)
    m2 = _FakeModel()
    res2 = speed.SpeedTester("cpu").test_speed(m2, list(speed.synthetic_items(1, False, 1, 16, 16, "cpu")), is_video=False)
    assert m2.calls[0] == ("embed", (1, 3, 16, 16), False, False) and m2.calls[1][0] == "detect"
    assert "avg_embedding_ms_per_frame" not in res2


def test_tensor_api_facade_forwards_to_the_model():
    """docs/torchscript.md surface: tuple / tensor returns, attribute plumbing, attenuation switch"""
    from videoseal_b200 import jit

    class M(_FakeModel):
        def __init__(self):
            super().__init__()
            self.blender = argparse.Namespace(scaling_w=0.2, scaling_i=1.0)
            self.img_size, self.clamp, self.chunk_size, self.step_size, self.video_mode = 256, True, 32, 4, "repeat"
            self.attenuation = "jnd_1_1"

    m = M()
    t = jit.TensorAPI(m)
    x = torch.rand(2, 3, 16, 16)
    img_w, preds = t(x, torch.zeros(2, 4))
    assert img_w.shape == x.shape and preds.shape == (2, 5)
    assert m.calls[0] == ("embed", (2, 3, 16, 16), False, True)          # lowres attenuation on by default, like the artefact
    assert t.chunk_size == 16 and m.chunk_size == 16
    t.scaling_w, t.step_size, t.video_mode, t.do_attenuation = 0.5, 8, "interpolate", False
    assert m.blender.scaling_w == 0.5 and m.step_size == 8 and m.video_mode == "interpolate" and m.attenuation is None
    t.do_attenuation = True
    assert m.attenuation == "jnd_1_1" and t.do_attenuation
    bits = t.detect_video_and_aggregate(x, aggregation="squared_avg")
    assert bits.dtype == torch.float32 and m.calls[-1] == ("extract", (2, 3, 16, 16), "squared_avg")


def test_streaming_loops_chunking_tail_and_thread_plumbing():
    """outer loops of the streaming CLI (inference_streaming.py:83-107,146-162) on in-memory RGB24 streams with stand-in clip functions"""
    import io
    import numpy as np
    from videoseal_b200 import streaming
    W, H, F_, CH = 6, 4, 11, 4
    rng = np.random.default_rng(0)
    frames = rng.integers(0, 256, (F_, H, W, 3), dtype=np.uint8)
    chunks = list(streaming.iter_rawvideo_chunks(io.BytesIO(frames.tobytes()), W, H, CH))
    assert [len(c) for c in chunks] == [4, 4, 3] and np.array_equal(np.concatenate(chunks), frames)
    assert list(streaming.iter_rawvideo_chunks(io.BytesIO(b""), W, H, CH)) == []

    class M:
        def get_random_msg(self):
            return torch.tensor([[1, 0, 1]])

    seen = []

    def fake_embed(model, clip, msgs):
        seen.append(len(clip))
        return 255 - clip

    dst = io.BytesIO()
    msgs = streaming.embed_stream(M(), io.BytesIO(frames.tobytes()), dst, W, H, CH, clip_fn=fake_embed)
    assert msgs.tolist() == [[1, 0, 1]] and seen == [4, 4, 3]
    assert np.array_equal(np.frombuffer(dst.getvalue(), np.uint8).reshape(F_, H, W, 3), 255 - frames)      # order and tail preserved

    def fake_detect(model, clip):
        return torch.from_numpy(clip.reshape(len(clip), -1)[:, :3].astype(np.float32))

    soft = streaming.detect_stream(M(), io.BytesIO(frames.tobytes()), W, H, CH, clip_fn=fake_detect)       # full chunks only, like the reference
    assert torch.allclose(soft, torch.from_numpy(frames[:8].reshape(8, -1)[:, :3].astype(np.float32)).mean(0))
    soft_all = streaming.detect_stream(M(), io.BytesIO(frames.tobytes()), W, H, CH, include_tail=True, clip_fn=fake_detect)
    assert torch.allclose(soft_all, torch.from_numpy(frames.reshape(F_, -1)[:, :3].astype(np.float32)).mean(0))
    with pytest.raises(ValueError):
        streaming.detect_stream(M(), io.BytesIO(frames[:3].tobytes()), W, H, CH, clip_fn=fake_detect)

    def boom(model, clip, msgs):
        raise RuntimeError("clip failed")

    with pytest.raises(RuntimeError, match="clip failed"):
        streaming.embed_stream(M(), io.BytesIO(frames.tobytes()), io.BytesIO(), W, H, CH, clip_fn=boom)
    import shutil
    if shutil.which("ffmpeg") is None:
        with pytest.raises(RuntimeError, match="ffmpeg"):
            streaming.embed_video(M(), "in.mp4", "out.mp4", 8)


def test_full_evaluation_slice_columns_and_values(tmp_path):
    """evals/full.py identity slice: the reference's column names, perfect decoding of a stand-in model that embeds nothing
    and returns the message as logits"""
    from videoseal_b200.evals import full

    class M:
        def __init__(self):
            self.msg = torch.tensor([[1, 0, 1, 1, 0, 0, 1, 0]])

        def embed(self, imgs, msgs=None, is_video=True, interpolation=None, lowres_attenuation=False):
            n = imgs.shape[0]
            return {"imgs_w": (imgs + 0.01).clamp(0, 1), "msgs": self.msg.repeat(n, 1)}

        def detect(self, imgs, is_video=True):
            z = self.msg.float() * 2 - 1
            return {"preds": torch.cat([torch.zeros(len(imgs), 1), z.repeat(len(imgs), 1)], 1)}

        def extract_message(self, imgs, aggregation="avg", interpolation=None):
            return self.msg.bool()

    items = list(speed.synthetic_items(2, True, 6, 16, 16, "cpu"))
    rows = full.evaluate(M(), items, True, str(tmp_path), num_frames=4)
    assert [r["iteration"] for r in rows] == [0, 1] and rows[0]["t"] == 6
    assert rows[0]["bit_acc_Identity_0"] == 1.0 and rows[0]["capacity_Identity_0"] == pytest.approx(8.0)
    assert rows[0]["pvalue_Identity_0"] == pytest.approx(0.5 ** 8) and rows[0]["log_pvalue_Identity_0"] == pytest.approx(8 * math.log10(2))
    assert 39.0 < rows[0]["psnr"] < 41.0                                  # +0.01 everywhere (minus clamping) ~ 40 dB
    lines = open(tmp_path / "metrics.csv").read().strip().splitlines()
    assert lines[0].split(",")[:5] == ["iteration", "t", "h", "w", "embed_time"] and len(lines) == 3
    rows_img = full.evaluate(M(), list(speed.synthetic_items(1, False, 1, 16, 16, "cpu")), False, str(tmp_path / "img"))
    assert rows_img[0]["bit_acc_Identity_0"] == 1.0 and rows_img[0]["t"] == 1


def test_checkpoint_loader_never_falls_back_to_the_full_unpickler(tmp_path):
    """ADVICE r1 (high): a checkpoint the safe unpickler rejects must raise, not execute"""
    import pickle
    from videoseal_b200 import cfg

    class Boom:
        def __reduce__(self):
            return (os.system, ("echo pwned > %s" % (tmp_path / "pwned"),))

    p = tmp_path / "evil.pth"
    torch.save({"args": Boom(), "model": {}}, p)
    with pytest.raises((pickle.UnpicklingError, RuntimeError, Exception)) as ei:
        cfg.get_config_from_checkpoint(str(p))
    assert not (tmp_path / "pwned").exists(), "the malicious reducer ran"
    assert "pwned" not in str(ei.value) or True


def test_embed_stream_surfaces_a_dead_writer_instead_of_deadlocking():
    """ADVICE r1 (medium): the encoder side dies on its 2nd (slow) write while the output queue is full"""
    import io
    import threading
    import time
    import numpy as np
    from videoseal_b200 import streaming

    w, h, cs, n = 8, 8, 2, 40
    src = io.BytesIO(np.zeros((n, h, w, 3), np.uint8).tobytes())

    class Dst:
        def __init__(self):
            self.n = 0

        def write(self, b):
            self.n += 1
            if self.n >= 2:
                time.sleep(0.3)
                raise BrokenPipeError("encoder went away")

    done = {}

    def run():
        try:
            streaming.embed_stream(None, src, Dst(), w, h, cs, msgs=torch.zeros(1, 4), prefetch=1, clip_fn=lambda m, c, ms: c)
        except BaseException as e:
            done["err"] = e

    t = threading.Thread(target=run, daemon=True)
    t.start()
    t.join(timeout=20)
    assert not t.is_alive(), "embed_stream deadlocked on a full queue with a dead writer"
    assert isinstance(done.get("err"), BrokenPipeError)


def test_baked_in_attributes_are_live_properties(built_lib):
    """ADVICE round 1 (low): img_size / embedder.yuv / attenuation are baked into the native handle; assigning them must
    rebuild it (or raise), never be a silent no-op (wam.py:147-149,196 mutate them freely in the reference)"""
    import videoseal_b200
    from videoseal_b200.model import JND
    from tests.util import synthetic_card_on_disk
    cpath, spec, _ = synthetic_card_on_disk("videoseal_1.0", tiny={"num_blocks": 1, "depths": [1, 1, 1, 1]})
    m = videoseal_b200.load(cpath).eval()
    assert m.img_size == spec["img_size"] == 256 and m.embedder.yuv is True
    m._native = None
    m.img_size = 384                                   # rebuilt lazily with the new processing size
    assert m.img_size == 384 and m.spec["img_size"] == 384 and m._native is None
    for bad in (0, 200, -128):
        with pytest.raises(ValueError):
            m.img_size = bad
    assert m.img_size == 384
    # attenuation: None switches it off; a JND with another channel layout re-specs the handle (jnd_1_1 -> jnd_3_3)
    assert m.attenuation is not None and tuple(m.spec["jnd"]) == (1, 1)
    keep = m.attenuation
    m.attenuation = None
    assert m.attenuation is None and tuple(m.spec["jnd"]) == (1, 1)
    m.attenuation = keep
    assert m.attenuation is keep

    class RefJND:                                      # duck-typed like the reference's modules/jnd.py object
        in_channels, out_channels = 3, 3
    m.attenuation = RefJND()
    assert isinstance(m.attenuation, JND) and tuple(m.spec["jnd"]) == (3, 3)
    with pytest.raises(ValueError):
        m.attenuation = object()
    # the Y-channel U-Net of this card cannot run on RGB input
    with pytest.raises(ValueError):
        m.embedder.yuv = False
    m.embedder.yuv = True
    # the tensor-API facade forwards to the same properties
    from videoseal_b200 import jit
    t = jit.TensorAPI(m) if hasattr(jit, "TensorAPI") else None
    if t is not None:
        t.img_size = 256
        assert m.img_size == 256
