"""-m gpu: the decoder against transformers' own OPTDecoderLayer stack run ON THE GPU under torch.autocast(fp16).

The unmodified reference cannot run here (flash-attn + transformers 4.39.3 + optimum + accelerate; SURVEY.md 8c), and
its arithmetic lives in those dependencies.  The closest executable stand-in for the reference's real arithmetic is
HF's `OPTDecoderLayer` (the class `ShapeOPTDecoder` stacks, shape_opt.py:205,403-410) with the synthetic checkpoint,
under the same autocast context `main.py` runs in (`accelerator.autocast()`, main.py:152), with SDPA attention
(fp16 in / fp32 accumulate, like flash-attn).  This pins the rounding points the CPU oracle mirrors -- fp16 Linear
outputs, fp32 LayerNorm and residual stream -- at FULL depth over 300 teacher-forced positions.
"""
import pytest
import torch

from tests.util import decoder_sd, random_prefix

gpu = pytest.mark.gpu
P = "transformer.model.decoder"


def _hf_autocast_logits(sd, n_layers, prefix, ids, dev):
    """fp16-autocast logits of every generated position, teacher-forced on `ids` (full-sequence recompute).
    Embeddings restated from shape_opt.py:237-245 (embed_with_vae), :318-337 (token / prefix embedding + cond_embed),
    :440-460 (OPTFacePositionalEmbedding) and modeling_opt.py:43-71 (learned positions, offset 2)."""
    from transformers import OPTConfig
    from transformers.models.opt.modeling_opt import OPTDecoderLayer
    cfg = OPTConfig(hidden_size=1024, num_hidden_layers=n_layers, ffn_dim=4096, num_attention_heads=16,
                    do_layer_norm_before=False, word_embed_proj_dim=1024, activation_function="relu",
                    enable_bias=True, layer_norm_elementwise_affine=True, dropout=0.0, attention_dropout=0.0)
    cfg._attn_implementation = "sdpa"
    g = lambda k: sd[k].to(dev)
    n = len(ids)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        rows = [prefix.to(dev) + g(f"{P}.cond_embed.weight")[0]]                       # shape_opt.py:331-337
        tok = torch.tensor(ids[:-1], device=dev)                                       # token fed at step i is ids[i-1]
        k = torch.arange(1, n, device=dev)                                             # tokens generated incl. current
        special = tok < 3
        x_code = torch.nn.functional.linear(g(f"{P}.quantize_codebooks")[0][(tok - 3).clamp(min=0)],
                                            g(f"{P}.input_layer.weight"), g(f"{P}.input_layer.bias"))   # fp16 (autocast)
        x = torch.where(special[:, None], g(f"{P}.extra_embeds.weight")[tok.clamp(max=2)], x_code.float())
        slot = torch.where(special, tok, (k - 2) % 9 + 3)                              # shape_opt.py:455-458
        e = x + g(f"{P}.token_embed_positions.weight")[slot] + g(f"{P}.cond_embed.weight")[1]
        emb = torch.cat(rows + [e], dim=0)[None]                                       # [1, 257+n-1, 1024] fp32
        S = emb.shape[1]
        hidden = emb + g(f"{P}.embed_positions.weight")[2:2 + S][None]                 # shape_opt.py:359-364
        causal = torch.full((S, S), float("-inf"), device=dev).triu(1)[None, None]
        for i in range(n_layers):
            layer = OPTDecoderLayer(cfg, layer_idx=i).eval().to(dev)
            layer.load_state_dict({kk[len(f"{P}.layers.{i}."):]: v for kk, v in sd.items()
                                   if kk.startswith(f"{P}.layers.{i}.")}, strict=True)
            out = layer(hidden, attention_mask=causal)
            hidden = out[0] if isinstance(out, tuple) else out
            del layer
        logits = torch.nn.functional.linear(hidden[0, 256:], g("transformer.lm_head.weight"))           # shape_opt.py:155
    return logits.float().cpu()                                                        # [n, vocab]


@gpu
@pytest.mark.slow
def test_decoder_vs_hf_autocast_fp16_full_depth():
    """24 layers, 300 teacher-forced positions (contexts 257..556, three attention chunks, special tokens included):
    fp16 logits of ma_decode_generate (default batch-1 greedy path: the per-phase kernels) vs HF OPTDecoderLayer x 24
    under fp16 autocast on the same GPU.  Tolerance: both sides round Linear outputs to fp16 but accumulate in different orders (cuBLAS / SDPA vs the
    canonical order), so individual activations can land on neighbouring fp16 values and the differences random-walk
    through 24 layers.  Asserted: max < 3e-2, mean < 3e-3, argmax equal wherever HF's top-2 margin exceeds
    4e-2 and at >= 99 % of all positions."""
    from meshanything_b200.decoder import DecoderArena, Generator
    dev = torch.device("cuda:0")
    NL, n = 24, 300
    sd = decoder_sd(NL)
    prefix = random_prefix(1, seed=4)
    arena = DecoderArena(sd, dev)
    gen = Generator(arena, 1, 257 + n)
    free, _ = gen.generate(prefix.to(dev), n, eos_id=-1)
    forced = free[0].cpu().tolist()
    for pos, t in ((5, 0), (6, 1), (7, 2), (100, 1), (255, 2), (256, 0)):
        forced[pos] = t
    f = torch.tensor([forced], dtype=torch.int32)
    ids, lens, logits = gen.generate(prefix.to(dev), n, forced_ids=f, want_logits=True, eos_id=-1)
    assert ids[0].cpu().tolist() == forced and int(lens[0]) == n   # every step ran and emitted its token
    got = logits[:, 0].cpu().float()
    ref = _hf_autocast_logits(sd, NL, prefix[0], forced, dev)
    diff = (got - ref).abs()
    top2 = torch.topk(ref, 2, dim=1).values
    margin = top2[:, 0] - top2[:, 1]
    agree = (got.argmax(1) == ref.argmax(1))
    print(f"decoder vs HF autocast fp16: max |diff| {float(diff.max()):.4f} mean {float(diff.mean()):.5f} "
          f"(logit std {float(ref.std()):.3f}); argmax agreement {float(agree.float().mean()):.4f} over {n} positions, "
          f"{int((margin > 0.1).sum())} with margin > 0.1")
    assert diff.max() < 3e-2 and diff.mean() < 3e-3
    clear = margin > 4e-2
    assert torch.equal(got.argmax(1)[clear], ref.argmax(1)[clear])
    assert agree.float().mean() >= 0.99
