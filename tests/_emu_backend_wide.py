"""TEST-ONLY: the emulation backend with CudaBackend's attention head-size limit (attn_max_head_dim = 256) and its
channel multiple of 32 (tests/_emu_backend_widths.py), plus the SpatialTransformer backward entry points of
tests/test_transformer_training_host.py.  Its attention methods are the oracle's, which take any head size; here they
check that the executors hand them only the sizes CudaBackend's kernels take.  The base EmuBackend declares no limit,
so the executors keep the 128 rule on it and its launch traces stay as they are."""
from _emu_backend_widths import EmuBackendWidths
from test_transformer_training_host import EmuBackend as _TransformerEmuBackend


def _check(C, heads):
    d = C // heads
    assert C % heads == 0 and d % 8 == 0 and 8 <= d <= 256, (C, heads)


class EmuBackendWide(EmuBackendWidths):
    attn_max_head_dim = 256
    layernorm_bwd = _TransformerEmuBackend.layernorm_bwd
    geglu_bwd = _TransformerEmuBackend.geglu_bwd

    def attention(self, qkv, heads, order, out_f32=None, out_hi=None, out_lo=None):
        _check(qkv.shape[-1] // 3, heads)
        super().attention(qkv, heads, order, out_f32, out_hi, out_lo)

    def attention_split(self, qkv_hi, qkv_lo, heads, order, out_f32=None, out_hi=None, out_lo=None):
        _check(qkv_hi.shape[-1] // 3, heads)
        super().attention_split(qkv_hi, qkv_lo, heads, order, out_f32, out_hi, out_lo)

    def attention_cross(self, q_hi, q_lo, kv_hi, kv_lo, heads, out_f32=None, out_hi=None, out_lo=None):
        _check(q_hi.shape[-1], heads)
        super().attention_cross(q_hi, q_lo, kv_hi, kv_lo, heads, out_f32, out_hi, out_lo)

    def attention_bwd(self, qkv, out, dout, heads, order, dqkv, lse, delta):
        _check(qkv.shape[-1] // 3, heads)
        super().attention_bwd(qkv, out, dout, heads, order, dqkv, lse, delta)

    def attention_cross_bwd(self, q, kv, out, dout, heads, dq, dkv, lse, delta):
        _check(q.shape[-1], heads)
        _TransformerEmuBackend.attention_cross_bwd(self, q, kv, out, dout, heads, dq, dkv, lse, delta)
