"""CPU: the MXFP8 scale-factor layout and quantisation rule, via the plain-PyTorch specification
(``ops/mx8.py::quantize_mx8_reference``) that the CUDA quantiser is tested against on the GPU."""
import torch

from bflc_demo_b200.ops.mx8 import SF_CHUNK, quantize_mx8_reference


def test_reference_quantizer_roundtrip_and_chunk_layout():
    torch.manual_seed(0)
    R, K = 300, 784
    x = torch.randn(R, K) * torch.logspace(-3, 2, K)
    m = quantize_mx8_reference(x)
    kb = (K + 127) // 128
    assert m.q.shape == (R, 784) and m.sf.numel() == ((R + 255) // 256 * 2) * kb * SF_CHUNK
    back = m.dequantize()
    rel = ((back - x).norm() / x.norm()).item()
    assert rel < 0.04                                     # e4m3 has 3 mantissa bits
    assert m.q.float().abs().max().item() <= 448.0
    # byte [r % 32][r // 32][k // 32] of chunk (row_block, k_block) is the scale of (row, group)
    r, g = 197, 13                                        # row 197 -> block 1, r0 = 5, r1 = 2
    chunk = (r // 128) * kb + g // 4
    byte = m.sf[chunk * SF_CHUNK + (r % 32) * 16 + ((r % 128) // 32) * 4 + g % 4].item()
    amax = x[r, g * 32:(g + 1) * 32].abs().max()
    want = next(e for e in range(3, 255) if 448.0 * 2.0 ** (e - 127) >= float(amax))   # exact
    assert byte == want
    # padding rows / groups carry scale 1.0
    assert m.sf[(((R + 255) // 256 * 2) - 1) * kb * SF_CHUNK + 31 * 16 + 3 * 4].item() == 127


def test_reference_quantizer_handles_u8_inputs_and_zero_groups():
    u = torch.zeros(128, 64, dtype=torch.uint8)
    u[:, :32] = torch.randint(1, 256, (128, 32), dtype=torch.uint8)
    m = quantize_mx8_reference(u, in_scale=1.0 / 255.0)
    back = m.dequantize()
    assert ((back - u.float() / 255.0).norm() / (u.float() / 255.0).norm()).item() < 0.04
    assert float(back[:, 32:].abs().sum()) == 0.0        # an all-zero group stays exactly zero
