"""The fragment-layout epilogues of the two kernels that run the generator's full-resolution launches, against float64
with the kernels' own rounding points at the bars of test_gpu_kernel_parity.py, in fp16 and bf16:

  * convt_fused_kernel (face_decoder_blocks.6.0, the 48x48 -> 96x96 transposed conv): scale / shift and ReLU on the
    accumulator fragment, one staging tile and TMA store per output phase, phases {00, 11} on one consumer warpgroup and
    {01, 10} on the other;
  * the row-major form of conv_patch_kernel (BN 16 and 32: output_block.0, the encoder's 16- and 32-channel blocks, the
    audio encoder, the K-folded first layers): scale / shift, the residual read from the patch centre and the activation
    on the fragment, and the fused 32 -> 3 head, whose dot products run in channel order after a butterfly inside each
    quad of lanes.

Every case asserts which kernel ran (w2l_debug_plan_kernels), runs twice with bit-identical results and leaves the fp16
range flag clear.  The tiles are ragged in both directions (W not a multiple of 8, H not a multiple of 16) and N is odd.
"""
import numpy as np
import pytest
import torch

import test_gpu_kernel_parity as P
from oracle import pipeline_oracle as PO
from oracle import w2l_oracle as O
from test_gpu_kernel_parity import BF16, F16, _c, _n, _t

pytestmark = pytest.mark.gpu

CASES = [
    # fused transposed conv (BK 32): 29 x 37 input = 4 x 3 tiles of 8 x 16, the last ones partly outside the image
    ("convT 160->64 ragged 29x37 N=3", _t(160, 64, 3, 2, 1, 1), 3, 37, 29, "T64.32"),
    ("convT 128->64 ragged 15x27 N=5", _t(128, 64, 3, 2, 1, 1), 5, 27, 15, "T64.32"),
    # row-major patch form, BN 16
    ("patch BN16 16 res ragged 29x45 N=3", _c(16, 16, 3, 1, 1, True), 3, 45, 29, "P16.16"),
    ("patch BN16 32->16 ragged 37x27 N=3", _c(32, 16, 3, 1, 1), 3, 27, 37, "P16.32"),
    # row-major patch form, BN 32
    ("patch BN32 32 res ragged 29x45 N=3", _c(32, 32, 3, 1, 1, True), 3, 45, 29, "P32.32"),
    ("patch BN32 48->32 ragged 37x27 N=3", _c(48, 32, 3, 1, 1), 3, 27, 37, "P32.16"),
    ("patch BN32 32 lrelu ragged 37x27 N=1", _n(32, 32, 3, 1, 1), 1, 27, 37, "P32.32"),
]


@pytest.fixture(scope="module", autouse=True)
def _contexts():
    yield
    for c in P._CTX.values():
        c.close()
    P._CTX.clear()


@pytest.mark.parametrize("prec", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_fullres_epilogue_matches_float64(case, prec):
    P.run_case(case, prec)


@pytest.mark.parametrize("prec", [F16, BF16], ids=["f16", "bf16"])
def test_generator_fullres_launches(prec):
    """face_decoder_blocks.6.0 stores its 64 channels into the first 64 channels of the 80-channel concat buffer, and
    output_block.0 carries the fused head: the generator at N = 3 checked layer by layer against float64 (and the head
    against the float64 sigmoid), twice, with bit-identical outputs and exported block outputs."""
    from wav2lip_b200 import _lib
    names = [n for n, _ in O.generator_layers()]
    i60 = names.index("face_decoder_blocks.6.0")
    runs = []
    for _ in range(2):
        out, ks, _worst = P._run_generator(prec, (), 3, slice(None))
        runs.append((out, P._export(P._ctx(prec), _lib.NET_GENERATOR, i60)))
    by_name = {}
    for k in ks:
        by_name.setdefault(k["name"].split(" ")[0], []).append(k)
    assert [P._short(k) for k in by_name["face_decoder_blocks.6.0"]] == ["T64.32"], by_name["face_decoder_blocks.6.0"]
    head = by_name["output_block.0"]
    assert [P._short(k) for k in head] == ["P32.16"] and head[0]["head"], head
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


def test_u8_head_is_truncated_fp32_head():
    """The uint8 form of the fused head stores trunc(__fmul_rn(s, 255)) of the same fp32 sigmoid the fp32 form stores:
    the uint8 path on uint8 crops equals the fp32 path on the same batch assembled on the host, times 255 in fp32,
    truncated.  N = 7 is odd."""
    from wav2lip_b200.models import Wav2Lip
    rng = np.random.RandomState(5)
    N = 7
    faces = rng.randint(0, 256, size=(N, 96, 96, 3), dtype=np.uint8)
    mels = (rng.rand(N, 80, 16).astype(np.float32) * 8 - 4)
    mel_b, img_b = PO.assemble_batch(faces, list(mels))
    g = Wav2Lip()
    g.load_state_dict(O.make_state_dict("generator", 0), strict=True)
    g = g.cuda().eval()
    with torch.no_grad():
        u8 = g.infer_u8(torch.from_numpy(mel_b).cuda(), torch.from_numpy(faces).cuda())
        y32 = g(torch.from_numpy(mel_b).cuda(), torch.from_numpy(img_b).cuda())
    expect = (y32.permute(0, 2, 3, 1) * torch.tensor(255.0, device=y32.device)).to(torch.uint8)
    assert u8.dtype == torch.uint8 and u8.shape == (N, 96, 96, 3)
    assert torch.equal(u8, expect), (u8.int() - expect.int()).abs().max().item()
