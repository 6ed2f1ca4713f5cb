"""Host side of the validation augmentations, without a GPU: the integer JPEG restatement equals PIL byte for byte, the random
parameter draws and column names equal the reference's (tests/golden/augment.pt), torchvision's grid parameters are restated
exactly, the C ABI is exported and its argument rules hold, and the codec rows raise."""
import io
import os

import numpy as np
import pytest
import torch
from PIL import Image

from tests.jpeg_oracle import jpeg_roundtrip
from videoseal_b200 import _lib
from videoseal_b200 import augmentation as A

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "augment.pt")


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN, weights_only=False)


def pil_jpeg(u8: np.ndarray, q: int) -> np.ndarray:
    b = io.BytesIO()
    Image.fromarray(u8).save(b, format="JPEG", quality=q)
    b.seek(0)
    return np.asarray(Image.open(b))


def _images():
    rng = np.random.default_rng(3)
    edge = np.zeros((40, 56, 3), np.uint8)
    edge[:, 23:] = 255
    edge[17:, :, 1] = 30
    ramp = np.linspace(0, 255, 50 * 70).reshape(50, 70)
    return {"random_45x61": rng.integers(0, 256, (45, 61, 3), dtype=np.uint8),
            "random_72x88": rng.integers(0, 256, (72, 88, 3), dtype=np.uint8),
            "random_odd_33x17": rng.integers(0, 256, (33, 17, 3), dtype=np.uint8),
            "flat": np.full((24, 40, 3), 173, np.uint8), "edge": edge,
            "ramp": np.stack([ramp, ramp[::-1], 255 - ramp], -1).astype(np.uint8),
            "tiny_3x4": rng.integers(0, 256, (3, 4, 3), dtype=np.uint8)}


@pytest.mark.parametrize("q", [40, 50, 60, 70, 80, 90])
def test_numpy_jpeg_equals_pil(q):
    for name, img in _images().items():
        got, want = jpeg_roundtrip(img, q), pil_jpeg(img, q)
        assert np.count_nonzero(got != want) == 0, name


def test_numpy_jpeg_equals_fixture(golden):
    for (k, q), want in golden["jpeg"].items():
        u8 = golden["inputs"][k][0].mul(255).byte().permute(1, 2, 0).numpy()
        assert np.count_nonzero(jpeg_roundtrip(u8, q) != want.numpy()) == 0, (k, q)


def test_parameter_draws_equal_the_reference(golden):
    x = golden["inputs"]["72x88"]
    for seed, d in golden["draws"].items():
        torch.manual_seed(seed)
        assert tuple(A.Crop().get_params(72, 88, 0.71)) == tuple(d["crop"])
        assert tuple(A.Crop(0.5, 0.9).get_params(72, 88)[2:]) == tuple(d["crop_random"])
        assert list(A.Perspective.get_perspective_params(88, 72, 0.5)) == list(d["perspective"])
        assert A.Perspective(0.1, 0.8).get_random_distortion_scale() == d["perspective_scale"]
        assert A.Rotate(5, 45).get_random_angle() == d["rotate"]
        assert tuple(A._random_size(0.5, 0.9, 72, 88)) == tuple(d["resize"])
        assert A.Brightness(0.5, 1.5).get_random_factor() == d["brightness"]
        assert A.JPEG(40, 90).get_random_quality() == d["jpeg"]
        assert A.GaussianBlur(3, 17).get_random_kernel_size() == d["blur"]
    assert x.shape == (1, 3, 72, 88)


def test_column_names_equal_the_reference(golden):
    for (is_video, oi, oc), names in golden["names"].items():
        if is_video and not oi:
            with pytest.raises(NotImplementedError):
                A.get_validation_augs(is_video, oi, oc)
            continue
        augs = A.get_validation_augs(is_video, oi, oc)
        assert [A.column_key(a, s) for a, ss in augs for s in ss] == names


def test_codec_rows_raise():
    for cls in (A.H264, A.H264rgb, A.H265, A.VP9, A.AV1):
        with pytest.raises(NotImplementedError):
            cls()(torch.zeros(1, 3, 8, 8), None, 30)
    with pytest.raises(NotImplementedError):
        A.Sequential(A.H264(), A.Crop(), A.Brightness())(torch.zeros(1, 3, 8, 8), None, (30, 0.71, 0.5))


def test_cpu_tensors_raise():
    with pytest.raises(RuntimeError, match="CUDA"):
        A.HorizontalFlip()(torch.zeros(1, 3, 8, 8), None, 0)


def test_torchvision_grid_parameters_are_restated_exactly():
    F = pytest.importorskip("torchvision.transforms.functional")
    from torchvision.transforms import _functional_tensor as FT
    for angle in (5, 10, 30, 45, 90, -90, 0, 17):
        assert A.inverse_affine_matrix(-angle) == F._get_inverse_affine_matrix([0.0, 0.0], -angle, [0.0, 0.0], 1.0, [0.0, 0.0])
        m = A.inverse_affine_matrix(-angle)
        for w, h in ((61, 45), (88, 72), (1920, 1080)):
            assert A.affine_output_size(m, w, h) == FT._compute_affine_output_size(m, w, h)
    torch.manual_seed(0)
    for scale in (0.1, 0.5, 0.8):
        start, end = A.Perspective.get_perspective_params(88, 72, scale)
        assert A.perspective_coeffs(start, end) == F._get_perspective_coeffs(start, end)
    for k in (3, 5, 9, 13, 17):
        sigma = 0.3 * ((k - 1) * 0.5 - 1) + 0.8
        assert A.gaussian_taps(k) == FT._get_gaussian_kernel1d(k, sigma, torch.float32, torch.device("cpu")).tolist()


def test_c_abi_is_exported_and_checks_arguments():
    L = _lib.lib()
    for name in ("vsb_augment", "vsb_augment_workspace_bytes"):
        assert name in _lib.EXPORTS and hasattr(L, name)
    assert L.vsb_augment_workspace_bytes(A.OPS["jpeg"], 2, 45, 61) >= 2 * 45 * 61 + 2 * 2 * 23 * 31
    assert L.vsb_augment_workspace_bytes(A.OPS["crop_flip"], 2, 45, 61) == 0
    assert L.vsb_augment_workspace_bytes(99, 2, 45, 61) < 0
    assert L.vsb_augment_workspace_bytes(A.OPS["blur"], 0, 45, 61) < 0
