"""TEST INFRASTRUCTURE ONLY — a torch restatement of the C-ABI operators the VAE encoder uses, so that engine.VaeEncoderEngine's
host side (conv_in's 8-channel operand, K64 weight packing, the end-padded stride-2 downsamplers, the mid block shared with
the decoder, quant_conv folded into conv_out) and AutoencoderKL.encode / encode_latents run in the build container against
oracle/vae_encode.py.  It installs every operator of tests/ops_emulator.py, then replaces `gemm_conv` with one that takes
K64-packed weights and end padding (include/magicdrive_b200.h: mdb_gemm_conv, pad_h_end / pad_w_end) and rejects keywords
it does not know, and `fid_input` with tests/fid_emulator.py's.  Activations stay fp32."""
import torch
import torch.nn.functional as F

from magicdrive_b200 import engine, models, ops
from tests import fid_emulator, ops_emulator


def gemm_conv(a0, w, *, n_img, h_in, w_in, c0, lda0, n_out, taps=1, stride=1, pad=0, pad_h_end=0, pad_w_end=0, bias=None,
              residual=None, ldr=0, out_f32=False, out_scale=1.0):
    """out = out_scale * (conv(F.pad(A, (pad, pad + pad_w_end, pad, pad + pad_h_end))) + bias) + residual."""
    assert pad_h_end >= 0 and pad_w_end >= 0, "negative end padding is rejected"
    k64 = (c0 + 63) // 64 * 64
    assert a0.stride(0) == lda0 and w.shape == (n_out, taps * taps * k64), (w.shape, n_out, taps, k64)
    wt = w.float().view(n_out, taps, taps, k64)
    assert torch.all(wt[..., c0:] == 0), "the K64 gap must hold zeros"
    x = a0[:, :c0].float().reshape(n_img, h_in, w_in, c0).permute(0, 3, 1, 2)
    y = F.conv2d(F.pad(x, (pad, pad + pad_w_end, pad, pad + pad_h_end)), wt[..., :c0].permute(0, 3, 1, 2), stride=stride)
    y = y.permute(0, 2, 3, 1).reshape(-1, n_out)
    if bias is not None:
        y = y + bias.float()
    y = y * out_scale
    if residual is not None:
        assert residual.stride(0) == ldr
        y = y + residual[:, :n_out].float()
    return y.contiguous() if out_f32 else ops_emulator._act(y)


def install(monkeypatch):
    ops_emulator.install(monkeypatch)
    monkeypatch.setattr(ops, "gemm_conv", gemm_conv)
    monkeypatch.setattr(ops, "fid_input", fid_emulator.fid_input)
    monkeypatch.setattr(engine._Weights, "fold_dtype", torch.float32)  # the quant_conv fold's algebra to fp32
    real = models.AutoencoderKL.encoder_engine

    def encoder_engine(self):  # the same checks, with the engine built on the CPU
        if self._encoder_missing or self._enc_engine is not None:
            return real(self)
        self._enc_engine = engine.VaeEncoderEngine(self.arch_cfg, dict(self.state_dict()), self.device)
        return self._enc_engine

    monkeypatch.setattr(models.AutoencoderKL, "encoder_engine", encoder_engine)
