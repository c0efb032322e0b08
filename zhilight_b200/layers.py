"""Host-side mirror of the reference's test-facing operator API `zhilight.internals_.layers`
(tests/py_export_internal/layer_linear.cpp:20-68): same constructor arguments, `load_state_dict`,
`named_parameters`, `forward`, so that a parity test reads like tests/test_linear.py:53-86.

`Linear` restates `nn::Linear`'s dispatch by QuantType (src/nn/linear/linear.cpp:1952-2075,
src/model/model_config.hpp:132-144): 0 Normal, 1/2 Int8 (2 = AutoInt8: quantise the fp weight at load,
linear.cpp:521-550), 5 GPTQ, 6 AWQ, 7 FP8, 8 GPTQ_Marlin (same checkpoint as 5, symmetric u4b8).
Every code path ends in the C-ABI (zhilight_b200.ops); there is no torch fallback -- without the CUDA library the
constructor raises."""
import torch

from . import _lib, ops

QUANT_NONE, QUANT_INT8, QUANT_AUTO_INT8, QUANT_GPTQ, QUANT_AWQ, QUANT_FP8, QUANT_GPTQ_MARLIN = 0, 1, 2, 5, 6, 7, 8
_DTYPES = {"half": torch.float16, "float16": torch.float16, "bfloat": torch.bfloat16, "bfloat16": torch.bfloat16}


class Linear:
    def __init__(self, dim_in, dim_out, activation="", quant=0, dtype="half", group_size=128, sym=False):
        _lib.load()                                      # fail loudly when the CUDA library is missing
        if dtype not in _DTYPES:
            raise ValueError("unknown dtype name %r" % dtype)
        self.dim_in, self.dim_out = int(dim_in), int(dim_out)
        self.activation = (activation or "").lower()
        if self.activation not in ("", "silu", "gelu"):
            raise ValueError("unsupported activation %r" % activation)
        self.quant = int(quant)                          # the reference's tests pass False for 0
        if self.quant not in (0, 1, 2, 5, 6, 7, 8):
            raise _lib.ZLError(-2, "quant value error: %d" % self.quant)
        self.dtype = _DTYPES[dtype]
        self.group_size, self.sym = group_size, bool(sym) or self.quant == QUANT_GPTQ_MARLIN
        if self.quant in (QUANT_GPTQ, QUANT_AWQ, QUANT_GPTQ_MARLIN) and self.dtype != torch.float16:
            raise _lib.ZLError(-2, "A must be half")     # q_gemm_k_major.cu:989
        self._p = {}
        self.bias = None

    # -- parameters -------------------------------------------------------------------------------------------
    def load_state_dict(self, state_dict):
        sd = {k: v.detach().cuda() for k, v in state_dict.items()}
        n, k = self.dim_out, self.dim_in
        self.bias = sd["bias"].to(self.dtype).contiguous() if "bias" in sd else None
        q = self.quant
        if q == QUANT_NONE:
            w = sd["weight"].to(self.dtype).contiguous()
            assert tuple(w.shape) == (n, k), "weight shape mismatch"
            self._p = {"weight": w}
        elif q in (QUANT_INT8, QUANT_AUTO_INT8):
            if q == QUANT_AUTO_INT8 or sd["weight"].dtype != torch.int8:
                wq, ws = ops.int8_quant_per_token(sd["weight"].to(self.dtype).contiguous())   # per output row
                ws = ws.to(self.dtype)                   # functions::typecast(w_scale, dtype), linear.cpp:541
            else:
                wq, ws = sd["weight"].contiguous(), sd["weight_scale"].to(self.dtype).contiguous()
            self._p = {"weight": wq, "weight_scale": ws}
        elif q == QUANT_FP8:
            w = sd["weight"]
            w = w.view(torch.uint8) if w.dtype != torch.uint8 else w
            self._p = {"weight": w.contiguous(), "weight_scale": sd["weight_scale"].float().reshape(1).contiguous()}
        else:
            is_awq = q == QUANT_AWQ
            g_idx = sd.get("g_idx")
            self._k_perm = None
            if g_idx is not None and not torch.equal(g_idx.cpu().int(),
                                                     (torch.arange(k) // self.group_size).int()):
                if q != QUANT_GPTQ:   # Marlin refuses act-order like the reference (linear.cpp:1418); AWQ has no g_idx
                    raise _lib.ZLError(-3, "act-order (desc_act) checkpoints are only supported with QuantType 5")
                qw, qz, sc, self._k_perm = ops.gptq_to_k_major_act_order(
                    sd["qweight"].int(), sd["qzeros"].int(), sd["scales"].half(), g_idx, self.group_size)
            else:
                qw, qz, sc = ops.gptq_to_k_major(sd["qweight"].int(), sd["qzeros"].int(), sd["scales"].half(), is_awq)
            self._p = {"qweight": qw, "qzeros": qz, "scales": sc}
            variant = 1 if _lib.load().zl_w4_int_kernel_fits(32, n, k) else 0
            self._packed = ops.w4_pack(qw, qz, sc, self.group_size, self.sym, None, variant)
            self._variant = variant

    def named_parameters(self):
        d = dict(self._p)
        if self.bias is not None:
            d["bias"] = self.bias
        return d

    # -- forward ----------------------------------------------------------------------------------------------
    def forward(self, x):
        if x.dim() not in (2, 3):
            raise _lib.ZLError(-1, "Input must be 2D")                    # linear.cpp:567
        if x.shape[-1] != self.dim_in:
            raise _lib.ZLError(-1, "Input size mismatch")
        if x.dtype != self.dtype:
            raise _lib.ZLError(-1, "Input data type mismatch")
        x2 = x.reshape(-1, self.dim_in).contiguous()
        q, n, k = self.quant, self.dim_out, self.dim_in
        if q == QUANT_NONE:
            y = ops.dense_gemm_skinny(x2, self._p["weight"], self.bias)
        elif q in (QUANT_INT8, QUANT_AUTO_INT8):
            y = ops.int8_linear(x2, self._p["weight"], self._p["weight_scale"], self.bias)
        elif q == QUANT_FP8:
            y = ops.fp8_linear(x2, self._p["weight"], self._p["weight_scale"], self.bias)
        else:
            kp = self._k_perm
            if kp is not None and not (self._variant == 1 and _lib.load().zl_w4_int_layout_route(x2.shape[0], n, k) == 3):
                x2, kp = ops.gather_cols(x2, kp), None   # only the integer kernel gathers while it stages x
            y = ops.w4a16_gemm_fused(x2, self._packed, n, k, self.group_size, bias=self.bias, variant=self._variant,
                                     k_perm=kp)
        if self.activation:
            y = ops.activation(y, self.activation)
        return y.reshape(*x.shape[:-1], n)

    __call__ = forward
