"""CPU oracle of a decode step over an int8 KV cache (the reference's KV_CACHE_DTYPE=int8).

Kv8OracleLlama is oracle.model.OracleLlama with every appended K (after RoPE) and V row quantised per (token, kv head)
by ops.int8_quant_per_token -- the quantisation oracle/check_golden.py pins against the reference's quant_calc_scale
(tests/golden/ref_kv8.npz) -- and attention run over the dequantised rows (code - 128) * scale.  The decode order is
OracleLlama.decode's; only the cache rows differ.
"""
import numpy as np

from oracle import model as omodel, ops

F32 = np.float32


def quant_rows(x):
    """(..., d) fp values -> uint8 codes (..., d) = int8 + 128 and fp32 scales (...): the cache contract."""
    x = np.asarray(x, F32)
    q, s = ops.int8_quant_per_token(x.reshape(-1, x.shape[-1]))
    return (q.astype(np.int32) + 128).astype(np.uint8).reshape(x.shape), s.reshape(x.shape[:-1])


def dequant_rows(codes, scales):
    return (np.asarray(codes, F32) - F32(128)) * np.asarray(scales, F32)[..., None]


class Kv8OracleLlama(omodel.OracleLlama):
    def __init__(self, *args, kv_int8=True, **kwargs):
        super().__init__(*args, **kwargs)
        self.kv_int8 = kv_int8
        self.codes = {}       # (task, layer) -> {position: (k codes, v codes, k scales, v scales)} of the appended rows

    def decode(self, tokens, positions, tasks=None):
        if not self.kv_int8:
            return super().decode(tokens, positions, tasks)
        c, T = self.c, self.dtype
        b = len(tokens)
        tasks = list(range(b)) if tasks is None else tasks
        d, hq, hkv = c["dim_head"], c["num_heads"], c["num_kv_heads"]
        h = omodel._f32(self.sd["token_embedding.weight"], T)[np.asarray(tokens)]
        cos, sin = ops.rope_cos_sin(np.asarray(positions), d, c["rope_theta"], c.get("rope_llama3"))
        scale = F32(1.0 / np.sqrt(d))
        for l in range(c["num_layers"]):
            p = "layers.%d." % l
            q, k, v = self._norm_linears(h, omodel._f32(self.sd[p + "ln_attn.weight"], T),
                                         [p + "attn.project_q", p + "attn.project_k", p + "attn.project_v"])
            q, k, v = ops.split_qkv_rope(np.concatenate([q, k, v], axis=1), cos, sin, hq, hkv, d, True, T)
            ao = np.zeros((b, hq * d), F32)
            for i, task in enumerate(tasks):
                kvs = self.kv.setdefault(task, [None] * c["num_layers"])
                if kvs[l] is None:
                    kvs[l] = (np.zeros((0, hkv, d), F32), np.zeros((0, hkv, d), F32))
                kb, vb = kvs[l]
                pos = int(positions[i])
                if kb.shape[0] <= pos:
                    pad = np.zeros((pos + 1 - kb.shape[0], hkv, d), F32)
                    kb, vb = np.concatenate([kb, pad]), np.concatenate([vb, pad])
                kc, ks = quant_rows(k[i].reshape(hkv, d))
                vc, vs = quant_rows(v[i].reshape(hkv, d))
                self.codes.setdefault((task, l), {})[pos] = (kc, vc, ks, vs)
                kb[pos] = dequant_rows(kc, ks)
                vb[pos] = dequant_rows(vc, vs)
                kvs[l] = (kb, vb)
                lb = pos + 1
                o = ops.decode_attention(q[i].reshape(1, 1, hq, d), [kb], [vb], [lb],
                                         [np.ones((1, lb), np.int8)], scale, hq // hkv, T)
                ao[i] = o.reshape(-1)
            h = ops.residual_add(h, self._linear(ao, p + "attn.attn_out"), T)
            g, u = self._norm_linears(h, omodel._f32(self.sd[p + "ln_ff.weight"], T), [p + "ff.w_in", p + "ff.w_gated"])
            h = ops.residual_add(h, self._linear(ops.silu_mul(g, u, T), p + "ff.w_out"), T)
        xn = ops.rmsnorm(h, omodel._f32(self.sd["output_layernorm.weight"], T), c["eps"], 1.0, T)
        lm = self.sd.get("lm_head.weight", self.sd["token_embedding.weight"])
        return np.asarray(xn, F32) @ omodel._f32(lm, T).T
