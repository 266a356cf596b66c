"""The engine pads the ViT MLP width to a multiple of 64 (4304 -> 4352, tiny 1008 -> 1024) with zero fc1 rows, zero fc1
bias and zero fc2 columns, so that the fc1 output and fc2's operands have 128-byte-aligned rows. The pad columns of the
fc1 output are exactly +0 and fc2 adds the same zeros TMA filled in before: results are unchanged bit for bit."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_mlp_width_padding_is_exact(dtype):
    """fc1 with 48 zero weight rows and zero bias writes exactly +0 in the pad columns; fc2 over the padded width equals
    fc2 over 4304 bit for bit (the same 68 k-blocks: TMA used to fill columns 4304.. with zeros)."""
    from visrag_b200 import ops

    M, D, H, HP = 8192, 1152, 4304, 4352
    g = torch.Generator(device="cuda").manual_seed(11)
    x = (torch.randn(M, D, device="cuda", generator=g) * 0.5).to(dtype)
    w1 = (torch.randn(H, D, device="cuda", generator=g) * 0.03).to(dtype)
    b1 = torch.randn(H, device="cuda", generator=g)
    w2 = (torch.randn(D, H, device="cuda", generator=g) * 0.03).to(dtype)
    b2 = torch.randn(D, device="cuda", generator=g)
    r = torch.randn(M, D, device="cuda", generator=g)
    w1p = torch.nn.functional.pad(w1, (0, 0, 0, HP - H))
    b1p = torch.nn.functional.pad(b1, (0, HP - H))
    w2p = torch.nn.functional.pad(w2, (0, HP - H))
    y = ops.gemm(x, w1, bias=b1, gelu=True)
    yp = ops.gemm(x, w1p, bias=b1p, gelu=True)
    torch.cuda.synchronize()
    assert torch.equal(yp[:, :H], y)
    pad = yp[:, H:].float()
    assert (pad == 0).all() and not torch.signbit(pad).any(), "pad columns must be exactly +0"
    z = r.clone()
    zp = r.clone()
    ops.gemm(y, w2, bias=b2, resid=z, out=z, out_dtype=torch.float32)
    ops.gemm(yp, w2p, bias=b2, resid=zp, out=zp, out_dtype=torch.float32)
    torch.cuda.synchronize()
    assert torch.equal(zp, z)


def _unpadded_vit_tokens(engine, pixels):
    """The engine's ViT with the MLP weights cut back to the model's width (what the engine ran before the padding)."""
    H = engine.cfg.vit_mlp
    saved = [(b["fc1_w"], b["fc1_b"], b["fc2_w"]) for b in engine.blocks]
    try:
        for b in engine.blocks:
            b["fc1_w"], b["fc1_b"], b["fc2_w"] = b["fc1_w"][:H].contiguous(), b["fc1_b"][:H].contiguous(), b["fc2_w"][:, :H].contiguous()
        return engine.vit_tokens(pixels)
    finally:
        for b, (w1, b1, w2) in zip(engine.blocks, saved):
            b["fc1_w"], b["fc1_b"], b["fc2_w"] = w1, b1, w2


@pytest.mark.parametrize("model", ["tiny", "full"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_engine_vit_tokens_equal_unpadded_width(model, dtype):
    """The engine's ViT tokens with the padded MLP width equal those with the model's width bit for bit."""
    from visrag_b200.config import VisRAGConfig
    from visrag_b200.encoder import VisRAGEngine
    from visrag_b200.weights import random_state_dict_device

    cfg = VisRAGConfig.tiny() if model == "tiny" else VisRAGConfig()
    sd = random_state_dict_device(cfg, 5, "cuda:0")
    eng = VisRAGEngine(cfg, sd, "cuda:0", dtype=dtype)
    assert eng.blocks[0]["fc1_w"].shape[0] % 64 == 0 and eng.blocks[0]["fc1_w"].shape[0] - cfg.vit_mlp < 64
    g = torch.Generator(device="cuda").manual_seed(1)
    S = 2 if model == "tiny" else 4
    pixels = torch.randint(0, 256, (S, 448, 448, 3), dtype=torch.uint8, device="cuda", generator=g)
    got = eng.vit_tokens(pixels)
    want = _unpadded_vit_tokens(eng, pixels)
    torch.cuda.synchronize()
    assert torch.isfinite(got.float()).all()
    assert torch.equal(got, want)
