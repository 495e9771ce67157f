"""Generate tests/golden/deepseek_v2_kat.pt: transformers' DeepSeek-V2 modules run on the CPU at the
tiny-deepseek-v2 shape, with the shape model's seeded weights.

transformers (5.5, `models/deepseek_v2/modeling_deepseek_v2.py`) is the definition of MLA attention,
the MoE block and the decoder layer.  This script builds `SynthModel('tiny-deepseek-v2', seed=0)`,
copies its weights into transformers' modules (per-expert linears into the fused `gate_up_proj` /
`down_proj`, the router's weight into `gate.weight`), and records on seeded inputs:
  attn      DeepseekV2Attention (sdpa) of layer 1 on x, with freqs_cis for the positions
  router    DeepseekV2Moe.route_tokens_to_experts of layer 1 on the fp32 logits: sel, fp32 weights
  moe       DeepseekV2Moe of layer 1 on x
  layer0/1  DeepseekV2DecoderLayer 0 (dense MLP) and 1 (MoE) on x
The rotary tables the shape model passes (fp32 cos / sin [S, 32]) are freqs_cis's real and imaginary
parts; both are stored.  The tests read the fixture only: they import neither transformers nor
anything outside the repository.

    python -m oracle.gen_deepseek_v2_golden
"""
import os

import torch

from llmc_b200.synth import SynthModel

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, '..', 'tests', 'golden', 'deepseek_v2_kat.pt')
B, S = 2, 37


def weight_digest(model):
    """A cheap fingerprint of the shape model's seeded weights: the fp64 sum of every parameter."""
    return {n: float(p.detach().double().sum()) for n, p in model.model.layers.named_parameters()}


@torch.no_grad()
def main():
    from transformers.models.deepseek_v2 import modeling_deepseek_v2 as hf
    from transformers import DeepseekV2Config

    torch.manual_seed(0)
    sm = SynthModel('tiny-deepseek-v2', seed=0)
    s = sm.shape
    cfg = DeepseekV2Config(
        vocab_size=s['vocab'], hidden_size=s['hidden'], intermediate_size=s['inter'],
        moe_intermediate_size=s['moe_inter'], num_hidden_layers=s['layers'], num_attention_heads=s['heads'],
        num_key_value_heads=s['heads'], n_routed_experts=s['experts'], n_shared_experts=s['shared_experts'],
        num_experts_per_tok=s['top_k'], first_k_dense_replace=s['first_k_dense'], kv_lora_rank=s['kv_lora'],
        q_lora_rank=None, qk_rope_head_dim=s['rope_dim'], qk_nope_head_dim=s['nope_dim'], v_head_dim=s['v_dim'],
        routed_scaling_factor=s['routed_scale'], topk_method='greedy', rms_norm_eps=s['rms_eps'],
        rope_parameters={'rope_type': 'default', 'rope_theta': s['rope_theta']},
        attn_implementation='sdpa', experts_implementation='eager')
    dt = s['dtype']

    layers = []
    for i, blk in enumerate(sm.model.layers):
        hl = hf.DeepseekV2DecoderLayer(cfg, i).to(dt).eval()
        sd = {}
        for n, p in blk.named_parameters():
            if '.experts.' in n:
                continue
            sd[n] = p.data
        if hasattr(blk.mlp, 'experts'):
            ex = blk.mlp.experts
            sd['mlp.experts.gate_up_proj'] = torch.stack(
                [torch.cat([e.gate_proj.weight, e.up_proj.weight]) for e in ex])
            sd['mlp.experts.down_proj'] = torch.stack([e.down_proj.weight for e in ex])
        missing, unexpected = hl.load_state_dict(sd, strict=False)
        assert not missing and not unexpected, (missing, unexpected)
        layers.append(hl)

    g = torch.Generator().manual_seed(7)
    x = torch.randn(B, S, s['hidden'], generator=g).to(dt)
    rot = hf.DeepseekV2RotaryEmbedding(cfg)
    pos_ids = torch.arange(S)[None].expand(B, S)
    freqs_cis = rot(x, pos_ids)                          # [B, S, 32] complex64
    cos, sin = freqs_cis[0].real.contiguous(), freqs_cis[0].imag.contiguous()

    attn = layers[1].self_attn(x, attention_mask=None, position_embeddings=freqs_cis)[0]
    moe_mod = layers[1].mlp
    logits = torch.nn.functional.linear(x.float(), moe_mod.gate.weight.float())
    sel, w = moe_mod.route_tokens_to_experts(logits)
    moe = moe_mod(x)
    out = {'x': x, 'cos': cos, 'sin': sin, 'attn': attn, 'sel': sel.reshape(B * S, -1), 'w': w.reshape(B * S, -1),
           'moe': moe, 'weights': weight_digest(sm)}
    for i, hl in enumerate(layers):
        out[f'layer{i}'] = hl(x, attention_mask=None, position_embeddings=freqs_cis)
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    torch.save(out, OUT)
    print('wrote', OUT, {k: tuple(v.shape) for k, v in out.items() if isinstance(v, torch.Tensor)})


if __name__ == '__main__':
    main()
