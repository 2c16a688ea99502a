"""
Same-box GPU reference timing (SURVEY.md section 8d): the reference's PyTorch GPU execution of the forward pass, rebuilt from
the library pieces the reference itself uses, timed beside the sm_90a path on identical weights and input.

  hac / fast : torch.nn.Conv1d + SiLU/tanh, torch.nn.LSTM (cuDNN, fp16) with flips, Linear + clamp -- the module tree
               bonito.nn builds with use_koi=False (bonito/nn.py:221-241,353-415,268-298).
  sup        : the host mirror's parameters driven through flash-attn's own kernels exactly as bonito/transformer/model.py:42-128
               does: RotaryEmbedding + flash_attn_qkvpacked_func(window), Triton rms_norm_fn with residual, swiglu, cuBLAS GEMMs.

Measurement aid, not part of the product path (and not a bench line): prints one JSON object per model.
"""
import argparse
import json
import os
import sys

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from bonito_b200 import synth  # noqa: E402


def timed(fn, steps, warmup):
    for _ in range(warmup):
        out = fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, out


def lstm_models(name, N, L):
    from bonito_b200.crf.model import Model
    from oracle.cpu_reference import CpuReferenceModel
    spec = synth.model_spec(name)
    weights = synth.make_weights(spec, seed=25)
    model = Model(synth.model_config(spec, batchsize=N, chunksize=L, overlap=0))
    model.load_state_dict(synth.state_dict_from_weights(spec, weights))
    model.use_koi(batchsize=N, chunksize=L, quantize=False)
    model = model.half().eval().cuda()
    ref = CpuReferenceModel(spec, weights).half().cuda()
    return model, (lambda x: ref(x).permute(1, 0, 2)), spec["state_len"]


def sup_models(N, L, depth):
    from bonito_b200.transformer import Model
    from bonito_b200.transformer import model as tm
    from bonito_b200.nn import LinearCRFEncoder
    spec = synth.sup_spec(depth=depth)
    sd = synth.sup_state_dict(spec, synth.make_sup_weights(spec, seed=25))
    model = Model(synth.sup_config(spec))
    model.load_state_dict(sd)
    model.use_koi(batchsize=N, chunksize=L, quantize=False)
    model = model.half().eval().cuda()

    ref = Model(synth.sup_config(spec))
    ref.load_state_dict(sd)

    def _no_blanks(m):      # blank-free scores like the native mode (reference: transformer/model.py:138-141)
        if isinstance(m, LinearCRFEncoder):
            m.expand_blanks = False
    ref.encoder.apply(_no_blanks)
    ref = ref.half().eval().cuda()

    from flash_attn import flash_attn_qkvpacked_func
    from flash_attn.layers.rotary import RotaryEmbedding
    from flash_attn.ops.activations import swiglu
    from flash_attn.ops.triton.layer_norm import rms_norm_fn
    rotary = {}

    def attn_forward(self, x):
        n, t, _ = x.shape
        qkv = self.Wqkv(x).view(n, t, 3, self.nhead, self.head_dim)
        if "r" not in rotary:
            rotary["r"] = RotaryEmbedding(self.rotary_dim, interleaved=False, device=x.device)
        qkv = rotary["r"](qkv)
        out = flash_attn_qkvpacked_func(qkv, window_size=self.attn_window)
        return self.out_proj(out.reshape(n, t, self.d_model))

    def norm_forward(self, x, residual=None):
        return rms_norm_fn(x, self.weight, None, residual=residual, eps=self.eps)

    def mlp_forward(self, x):
        y, gate = self.fc1(x).chunk(2, dim=-1)
        return self.fc2(swiglu(gate, y))

    for m in ref.modules():
        if isinstance(m, tm.MultiHeadAttention):
            m.forward = attn_forward.__get__(m)
        elif isinstance(m, tm.RMSNorm):
            m.forward = norm_forward.__get__(m)
        elif isinstance(m, tm.GatedMlp):
            m.forward = mlp_forward.__get__(m)
    return model, (lambda x: ref.encoder(x).permute(1, 0, 2)), spec["state_len"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="hac", choices=["fast", "hac", "sup"])
    ap.add_argument("--batch", type=int, default=None)
    ap.add_argument("--chunk", type=int, default=9996)
    ap.add_argument("--depth", type=int, default=18)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    N = args.batch or (256 if args.model == "sup" else 512)
    L = args.chunk
    if args.model == "sup":
        model, ref_fwd, k = sup_models(N, L, args.depth)
    else:
        model, ref_fwd, k = lstm_models(args.model, N, L)
    x = synth.squiggle(32, L, seed=1).repeat(N // 32 + 1, 1, 1)[:N].half().cuda()
    out = {"model": args.model, "batch": N, "chunk": L}
    with torch.inference_mode():
        ms_nat, s_nat = timed(lambda: model(x), args.steps, args.warmup)
        out["native_forward_ms"] = ms_nat
        out["native_forward_samples_per_s"] = N * L / (ms_nat * 1e-3)
        try:
            ms_ref, s_ref = timed(lambda: ref_fwd(x), args.steps, args.warmup)
            out["torch_gpu_forward_ms"] = ms_ref
            out["torch_gpu_forward_samples_per_s"] = N * L / (ms_ref * 1e-3)
            out["speedup_forward"] = ms_ref / ms_nat
            d = (s_nat.float() - s_ref.float()).abs()
            out["scores_max_abs_diff"] = d.max().item()
            out["scores_mean_abs_diff"] = d.mean().item()
        except Exception as exc:  # library kernel unavailable on this box: report, do not hide
            out["torch_gpu_error"] = f"{type(exc).__name__}: {exc}"[:300]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
