"""Two models of one checkpoint on two GPUs in one process.  The kernels that use more than 48 KB of shared memory must be allowed
it on each device, since that limit is a per-device attribute: the same embed and detect run on cuda:0, then cuda:1, then
cuda:0 again, and the outputs are bit-identical across devices (the path is deterministic, DESIGN.md §4).  The 300 x 400 frames
reach the resize kernel and both blend kernels."""
import pytest
import torch

from tests.util import make_model_pair

pytestmark = pytest.mark.gpu


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_devices_one_process():
    pairs = [make_model_pair("videoseal_1.0", device=f"cuda:{d}") for d in (0, 1)]
    nbits = pairs[0][2]["nbits"]
    g = torch.Generator().manual_seed(0)
    cases = [(torch.rand(3, 3, H, W, generator=g), torch.randint(0, 2, (3, nbits), generator=g)) for H, W in ((256, 256), (300, 400))]
    first = {}
    for dev in (0, 1, 0):
        model = pairs[dev][0]
        for i, (imgs, msgs) in enumerate(cases):
            out = model.embed(imgs.to(f"cuda:{dev}"), msgs, is_video=False)
            det = model.detect(out["imgs_w"], is_video=False)["preds"]
            got = (out["imgs_w"].cpu(), det.cpu())
            if i not in first:
                first[i] = got
                continue
            assert torch.equal(got[0], first[i][0]), f"imgs_w of {tuple(imgs.shape)} differs on cuda:{dev}"
            assert torch.equal(got[1], first[i][1]), f"logits of {tuple(imgs.shape)} differ on cuda:{dev}"
