"""-m gpu: the staged chunk merge of attention_kernel (prefill, and decode at batch 1) against the oracle, bit for bit."""
import pytest
import torch

gpu = pytest.mark.gpu


@gpu
@pytest.mark.parametrize("H,T,nk", [(16, 7459, [1, 255, 256, 257, 1023, 1024, 1025, 7459]),
                                    (1, 64000, [63489, 63488, 64000])])
def test_attention_merge_bit_exact(H, T, nk):
    """One query row per nkeys.  7459 keys = the longest context of an 800-face generate; 63489 keys = 249 chunks,
    more partials than one staging round of the merge holds."""
    from meshanything_b200 import capi
    from oracle import decoder as orc
    g = torch.Generator().manual_seed(T + H)
    M = len(nk)
    q = torch.randn(M, H, 64, generator=g).half()
    k = torch.randn(H, T, 64, generator=g).half()
    v = torch.randn(H, T, 64, generator=g).half()
    ref = orc.attention(q, k, v, nk)
    d = torch.device("cuda:0")
    slots = torch.zeros(M, dtype=torch.int32, device=d)
    nkeys = torch.tensor(nk, dtype=torch.int32, device=d)
    got = capi.attention_f16(q.to(d), k.unsqueeze(0).contiguous().to(d), v.unsqueeze(0).contiguous().to(d), nkeys,
                             slots).cpu()
    assert torch.equal(got.view(torch.int16), ref.view(torch.int16))
