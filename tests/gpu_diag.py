"""GPU diagnostic runner (not a pytest file): runs every conv/GEMM unit case in its own subprocess (a trapped kernel
poisons the CUDA context) with a timeout, then a layer-by-layer parity walk of the whole network against the oracle.
Usage on the GPU box:  python tests/gpu_diag.py [--cases a,b] [--skip-net]  -> gpurun_out/diag.jsonl"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def one_case(name):
    import torch  # noqa
    from tests.conv_cases import run_case
    res = run_case(name, verbose=True)
    print("RESULT " + json.dumps({"case": name, **res}))


def net_walk(card):
    import torch
    from tests.util import make_model_pair
    tiny = None
    if card.endswith(":tiny"):      # chunkyseal:tiny = every width / map size of the card, reduced depth (tests/test_e2e_gpu.py)
        card, tiny = card[:-5], {"num_blocks": 1, "depths": [1, 1, 2, 1]}
    model, orc, spec = make_model_pair(card, device="cuda:0", tiny=tiny)
    g = torch.Generator().manual_seed(0)
    B = 2
    imgs = torch.rand(B, 3, 256, 256, generator=g)
    msgs = torch.randint(0, 2, (B, spec["nbits"]), generator=g)
    taps = {}
    ref_delta = orc.embedder(imgs, msgs, taps)
    rows = []

    def cmp(name, ref_nchw):
        try:
            got = model.debug_tensor(name)
        except Exception as e:
            rows.append({"tensor": name, "error": str(e)})
            return
        if name == "delta":
            g_ = got
        else:
            g_ = got.permute(0, 3, 1, 2)
        ref = ref_nchw
        if g_.shape != ref.shape:
            rows.append({"tensor": name, "shape_got": list(g_.shape), "shape_ref": list(ref.shape)})
            return
        err = (g_ - ref).abs()
        rows.append({"tensor": name, "maxerr": err.max().item(), "ref_absmax": ref.abs().max().item(),
                     "meanerr": err.mean().item(), "nan": int(torch.isnan(g_).sum())})

    ref = orc.embed(imgs, msgs, is_video=False)
    try:
        out = model.embed(imgs.cuda(), msgs, is_video=False)
        torch.cuda.synchronize()
        nd = len(spec["unet"]["mults"]) - 1
        for i in range(nd - 1):
            cmp(f"down{i}", taps[f"down{i}"])
        for i in range(spec["unet"]["num_blocks"]):
            cmp(f"bott{i}", taps[f"bott{i}"])
        for j in range(nd):
            cmp(f"up{j}_conv", taps[f"up{j}_conv"])
            if j < nd - 1:
                cmp(f"up{j}", taps[f"up{j}"])
        cmp("delta", ref_delta)
        rows.append({"tensor": "imgs_w", "maxerr": (out["imgs_w"].cpu() - ref["imgs_w"]).abs().max().item()})
        rows.append({"tensor": "preds_w", "maxerr": (out["preds_w"].cpu() - ref["preds_w"]).abs().max().item()})
    except Exception as e:   # keep going: the extractor walk below does not depend on the embedder
        rows.append({"tensor": "embed", "error": repr(e)[:1500]})
    for r in rows:
        print("RESULT " + json.dumps({"card": card, **r}), flush=True)
    rows.clear()
    # extractor on the ORACLE's watermarked image so errors do not compound
    taps = {}
    ref_logits = orc.detector(ref["imgs_w"], taps)
    got_logits = model.detect(ref["imgs_w"].cuda(), is_video=False)["preds"].cpu()
    # per-block kernels are judged on their own inputs by tests/test_cnx_kernels_gpu.py
    for s in range(4):
        cmp(f"stage{s}", taps[f"stage{s}"])
    err = (got_logits - ref_logits).abs()
    rows.append({"tensor": "logits", "maxerr": err.max().item(), "ref_absmax": ref_logits.abs().max().item(),
                 "bit_mismatch": int(((got_logits[:, 1:] > 0) != (ref_logits[:, 1:] > 0)).sum())})
    for r in rows:
        print("RESULT " + json.dumps({"card": card, **r}))


def main():
    args = sys.argv[1:]
    if args and args[0] == "--one":
        return one_case(args[1])
    if args and args[0] == "--net":
        return net_walk(args[1])
    from tests.conv_cases import CASES
    cases = list(CASES)
    skip_net = "--skip-net" in args
    net_card = "videoseal_1.0"
    for i, a in enumerate(args):
        if a == "--net-card":
            net_card = args[i + 1]
    for i, a in enumerate(args):
        if a == "--cases":
            cases = args[i + 1].split(",")
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    log = open(os.path.join(ROOT, "gpurun_out", "diag.jsonl"), "a")

    def run(cmd, tag, timeout):
        t0 = time.time()
        try:
            p = subprocess.run([sys.executable, os.path.abspath(__file__)] + cmd, capture_output=True, text=True, timeout=timeout)
            lines = [l[7:] for l in p.stdout.splitlines() if l.startswith("RESULT ")]
            if not lines:
                lines = [json.dumps({"case": tag, "ok": False, "rc": p.returncode, "stderr": p.stderr[-1500:]})]
        except subprocess.TimeoutExpired:
            lines = [json.dumps({"case": tag, "ok": False, "timeout": timeout})]
        for l in lines:
            print(f"[{time.time()-t0:5.1f}s] {l[:600]}", flush=True)
            log.write(l + "\n")
            log.flush()

    if "--no-cases" in args:
        cases = []
    for c in cases:
        run(["--one", c], c, 180)
    if not skip_net:
        run(["--net", net_card], "net:" + net_card, 600)


if __name__ == "__main__":
    main()
