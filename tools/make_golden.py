#!/usr/bin/env python
"""Generate tests/golden/*.npz — the committed golden vectors of the CPU oracle — and pin the oracle independently.

The reference ships no golden vectors (SURVEY §4/§8c: parity unpinned), and its arithmetic (ggml/llama.cpp) is not on
disk, so the goldens are (1) outputs of the oracle on seeded tiny models, re-creatable bit for bit from the seeds, and
(2) an INDEPENDENT float cross-check of the oracle's wiring against HuggingFace transformers' Blip2VisionModel /
Blip2QFormerModel / LlamaForCausalLM (fp32, same synthetic weights) — not the parity target, a sanity pin whose
measured deviations are stored in golden/crosscheck.json and asserted by tests/test_golden.py.

Run here (CPU):  python tools/make_golden.py            (transformers is needed only for the cross-check part)
"""
from __future__ import annotations

import json
import sys
import tempfile
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from minigpt4_cpp_b200 import modelgen as mg  # noqa: E402
from oracle import oracle as orc  # noqa: E402

GOLD = ROOT / "tests" / "golden"
TEXTS = ["Human: <Img>", "</Img> ", "### Assistant:", "what is this?", "héllo wörld ✓", "Give the following image: <Img>ImageContent</Img>."]
TOKENS = [1, 266, 61, 35, 63, 316, 65, 17, 900, 511, 3, 258, 700]
LONG_TOKENS = 2048   # the long cross-check: the F16 model over a whole n_ctx 2048 context

VISION_SPEC = dict(n_blocks=2, n_qformer_layers=2, n_embd_llm=4096)
LLAMA_SPECS = {
    "q4_1": dict(n_vocab=1024, n_embd=512, n_head=4, n_layer=2, wtype="q4_1"),
    "q4_0": dict(n_vocab=1024, n_embd=512, n_head=4, n_layer=2, wtype="q4_0"),
    "q5_k": dict(n_vocab=1024, n_embd=512, n_head=4, n_layer=2, wtype="q5_k"),
    "q6_k": dict(n_vocab=1024, n_embd=512, n_head=4, n_layer=2, wtype="q6_k"),
    "f16": dict(n_vocab=1024, n_embd=512, n_head=4, n_layer=2, wtype="f16"),
}


def oracle_goldens(d: Path):
    out = {}
    vis = d / "vision.bin"
    mg.write_minigpt4(vis, mg.VisionSpec(**VISION_SPEC))
    e = orc.OracleEngine(str(vis), None)
    img = mg.synth_image()
    emb = e.encode_image(img)
    out["vision_embedding"] = emb.astype(np.float32)
    out["vision_ln_vision_row0"] = e.encode_image(img, tap_kind=3)[0].astype(np.float32)
    out["vision_block0_row5"] = e.encode_image(img, tap_kind=2, tap_idx=0)[5].astype(np.float32)
    for name, spec in LLAMA_SPECS.items():
        p = d / f"llama-{name}.bin"
        mg.write_llama_ggjt(p, mg.LlamaSpec(**spec))
        e = orc.OracleEngine(None, str(p), n_ctx=128)
        e.eval_tokens(TOKENS)
        out[f"llama_{name}_logits"] = e.logits.copy()
        out[f"llama_{name}_greedy"] = np.array([e.end_chat_greedy()[0] for _ in range(16)], np.int32)
        if name == "q4_1":
            for i, t in enumerate(TEXTS):
                out[f"tok_{i}"] = np.array(e.tok.tokenize(t, True), np.int32)
    np.savez_compressed(GOLD / "oracle_golden.npz", **out)
    print("wrote", GOLD / "oracle_golden.npz", {k: v.shape for k, v in out.items() if k.startswith("vision")})


def crosscheck_transformers(d: Path) -> dict:
    import torch
    from transformers import Blip2QFormerConfig, Blip2QFormerModel, Blip2VisionConfig, Blip2VisionModel, LlamaConfig, LlamaForCausalLM
    torch.set_grad_enabled(False)
    res = {}
    # ---------------- vision tower + Q-Former ----------------
    vis = d / "vision.bin"
    _, T = orc.read_minigpt4(str(vis))

    def f32(name):
        t = T[name]
        a = np.frombuffer(t.data, np.float16 if t.gtype == 1 else np.float32).astype(np.float32)
        return torch.from_numpy(a.reshape(t.ne[::-1]).copy())

    vc = Blip2VisionConfig(hidden_size=1408, intermediate_size=6144, num_hidden_layers=VISION_SPEC["n_blocks"], num_attention_heads=16, image_size=224,
                           patch_size=14, hidden_act="gelu_pytorch_tanh", layer_norm_eps=1e-5, qkv_bias=True)
    vm = Blip2VisionModel(vc).eval().float()
    sd = {}
    sd["embeddings.class_embedding"] = f32("visual_encoder.cls_token").reshape(1, 1, -1)
    sd["embeddings.position_embedding"] = f32("visual_encoder.pos_embed").reshape(1, 257, -1)
    sd["embeddings.patch_embedding.weight"] = f32("visual_encoder.patch_embed.proj.weight")
    sd["embeddings.patch_embedding.bias"] = f32("visual_encoder.patch_embed.proj.bias")
    for i in range(VISION_SPEC["n_blocks"]):
        p, q = f"visual_encoder.blocks.{i}.", f"encoder.layers.{i}."
        sd[q + "self_attn.qkv.weight"] = f32(p + "attn.qkv.weight")
        qkv_bias = torch.cat([f32(p + "attn.q_bias"), torch.zeros(1408), f32(p + "attn.v_bias")])
        sd[q + "self_attn.projection.weight"] = f32(p + "attn.proj.weight"); sd[q + "self_attn.projection.bias"] = f32(p + "attn.proj.bias")
        sd[q + "layer_norm1.weight"] = f32(p + "norm1.weight"); sd[q + "layer_norm1.bias"] = f32(p + "norm1.bias")
        sd[q + "layer_norm2.weight"] = f32(p + "norm2.weight"); sd[q + "layer_norm2.bias"] = f32(p + "norm2.bias")
        sd[q + "mlp.fc1.weight"] = f32(p + "mlp.fc1.weight"); sd[q + "mlp.fc1.bias"] = f32(p + "mlp.fc1.bias")
        sd[q + "mlp.fc2.weight"] = f32(p + "mlp.fc2.weight"); sd[q + "mlp.fc2.bias"] = f32(p + "mlp.fc2.bias")
        keys = dict(vm.state_dict()).keys()
        if q + "self_attn.qkv.bias" in keys:
            sd[q + "self_attn.qkv.bias"] = qkv_bias
        else:
            sd[q + "self_attn.q_bias"] = f32(p + "attn.q_bias"); sd[q + "self_attn.v_bias"] = f32(p + "attn.v_bias")
    sd["post_layernorm.weight"] = f32("ln_vision.weight"); sd["post_layernorm.bias"] = f32("ln_vision.bias")
    missing, unexpected = vm.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    img = mg.synth_image()
    hf = vm(pixel_values=torch.from_numpy(img)[None]).last_hidden_state[0].numpy()  # = ln_vision(ViT(x)) (post_layernorm on all tokens)
    e = orc.OracleEngine(str(vis), None)
    mine = e.encode_image(img, tap_kind=3)
    res["vision_ln_vision_rel_err"] = float(np.abs(hf - mine).max() / np.abs(hf).max())
    res["vision_missing_keys"] = sorted(missing)

    qc = Blip2QFormerConfig(hidden_size=768, num_hidden_layers=VISION_SPEC["n_qformer_layers"], num_attention_heads=12, intermediate_size=3072,
                            hidden_act="gelu_pytorch_tanh", layer_norm_eps=1e-5, cross_attention_frequency=2, encoder_hidden_size=1408, vocab_size=30523,
                            hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    qm = Blip2QFormerModel(qc).eval().float()
    qsd = {"layernorm.weight": f32("Qformer.bert.embeddings.LayerNorm.weight"), "layernorm.bias": f32("Qformer.bert.embeddings.LayerNorm.bias")}
    for i in range(VISION_SPEC["n_qformer_layers"]):
        p, q = f"Qformer.bert.encoder.layer.{i}.", f"encoder.layer.{i}."
        for att, hatt in (("attention", "attention"), ("crossattention", "crossattention")):
            if p + att + ".self.query.weight" not in T:
                continue
            for nm in ("query", "key", "value"):
                qsd[q + f"{hatt}.attention.{nm}.weight"] = f32(p + f"{att}.self.{nm}.weight"); qsd[q + f"{hatt}.attention.{nm}.bias"] = f32(p + f"{att}.self.{nm}.bias")
            qsd[q + f"{hatt}.output.dense.weight"] = f32(p + f"{att}.output.dense.weight"); qsd[q + f"{hatt}.output.dense.bias"] = f32(p + f"{att}.output.dense.bias")
            qsd[q + f"{hatt}.output.LayerNorm.weight"] = f32(p + f"{att}.output.LayerNorm.weight"); qsd[q + f"{hatt}.output.LayerNorm.bias"] = f32(p + f"{att}.output.LayerNorm.bias")
        qsd[q + "intermediate_query.dense.weight"] = f32(p + "intermediate_query.dense.weight"); qsd[q + "intermediate_query.dense.bias"] = f32(p + "intermediate_query.dense.bias")
        qsd[q + "output_query.dense.weight"] = f32(p + "output_query.dense.weight"); qsd[q + "output_query.dense.bias"] = f32(p + "output_query.dense.bias")
        qsd[q + "output_query.LayerNorm.weight"] = f32(p + "output_query.LayerNorm.weight"); qsd[q + "output_query.LayerNorm.bias"] = f32(p + "output_query.LayerNorm.bias")
    missing, unexpected = qm.load_state_dict(qsd, strict=False)
    assert not unexpected, unexpected
    qtok = f32("query_tokens.weight").reshape(1, 32, 768)
    enc = torch.from_numpy(mine)[None]
    hq = qm(query_embeds=qtok, encoder_hidden_states=enc, encoder_attention_mask=torch.ones(1, 257, dtype=torch.long)).last_hidden_state[0]
    proj = hq @ f32("llama_proj.weight").T + f32("llama_proj.bias")
    mine_emb = e.encode_image(img)
    res["qformer_proj_rel_err"] = float(np.abs(proj.numpy() - mine_emb).max() / np.abs(proj.numpy()).max())
    res["qformer_missing_keys"] = sorted(k for k in missing if "intermediate." not in k and "output.dense" not in k and "output.LayerNorm" not in k)

    # ---------------- LLaMA (dequantised weights, float activations) ----------------
    for name in ("q4_1", "f16"):
        spec = mg.LlamaSpec(**LLAMA_SPECS[name])
        p = d / f"llama-{name}.bin"
        hp, _, LT = orc.read_ggjt(str(p))
        E, H = spec.n_embd, spec.n_head

        def W(nm):
            t = LT[nm]
            if len(t.ne) == 1:
                return torch.from_numpy(np.frombuffer(t.data, np.float32).copy())
            return torch.from_numpy(mg.dequant(t.gtype, np.frombuffer(t.data, np.uint8).reshape(t.ne[1], -1), t.ne[0]).copy())

        def permute(w):  # ggml/Meta adjacent-pair RoPE layout -> HF rotate_half layout
            return w.view(H, E // H // 2, 2, E).transpose(1, 2).reshape(E, E)

        lc = LlamaConfig(vocab_size=spec.n_vocab, hidden_size=E, intermediate_size=spec.n_ff, num_hidden_layers=spec.n_layer, num_attention_heads=H,
                         num_key_value_heads=H, rms_norm_eps=1e-6, rope_theta=10000.0, max_position_embeddings=LONG_TOKENS, tie_word_embeddings=False, attention_bias=False)
        lm = LlamaForCausalLM(lc).eval().float()
        lsd = {"model.embed_tokens.weight": W("tok_embeddings.weight"), "model.norm.weight": W("norm.weight"), "lm_head.weight": W("output.weight")}
        for i in range(spec.n_layer):
            a, b = f"layers.{i}.", f"model.layers.{i}."
            lsd[b + "self_attn.q_proj.weight"] = permute(W(a + "attention.wq.weight")); lsd[b + "self_attn.k_proj.weight"] = permute(W(a + "attention.wk.weight"))
            lsd[b + "self_attn.v_proj.weight"] = W(a + "attention.wv.weight"); lsd[b + "self_attn.o_proj.weight"] = W(a + "attention.wo.weight")
            lsd[b + "mlp.gate_proj.weight"] = W(a + "feed_forward.w1.weight"); lsd[b + "mlp.down_proj.weight"] = W(a + "feed_forward.w2.weight")
            lsd[b + "mlp.up_proj.weight"] = W(a + "feed_forward.w3.weight")
            lsd[b + "input_layernorm.weight"] = W(a + "attention_norm.weight"); lsd[b + "post_attention_layernorm.weight"] = W(a + "ffn_norm.weight")
        missing, unexpected = lm.load_state_dict(lsd, strict=False)
        assert not unexpected and not [m_ for m_ in missing if "rotary" not in m_], (missing, unexpected)
        hf_logits = lm(torch.tensor([TOKENS])).logits[0, -1].numpy()
        e = orc.OracleEngine(None, str(p), n_ctx=128)
        e.eval_tokens(TOKENS)
        res[f"llama_{name}_logits_rel_err"] = float(np.abs(hf_logits - e.logits).max() / np.abs(hf_logits).max())
        res[f"llama_{name}_argmax_equal"] = bool(int(np.argmax(hf_logits)) == int(np.argmax(e.logits)))
        if name == "f16":   # a whole 2048-token context: RoPE, attention and the soft-max sum up to the last position
            ids = np.random.default_rng(LONG_TOKENS).integers(3, spec.n_vocab, size=LONG_TOKENS)
            hf_logits = lm(torch.from_numpy(ids)[None]).logits[0, -1].numpy()
            e = orc.OracleEngine(None, str(p), n_ctx=LONG_TOKENS)
            e.eval_tokens(ids.tolist())
            res["llama_f16_long_logits_rel_err"] = float(np.abs(hf_logits - e.logits).max() / np.abs(hf_logits).max())
            res["llama_f16_long_argmax_equal"] = bool(int(np.argmax(hf_logits)) == int(np.argmax(e.logits)))
    return res


def main():
    GOLD.mkdir(parents=True, exist_ok=True)
    with tempfile.TemporaryDirectory() as td:
        d = Path(td)
        oracle_goldens(d)
        try:
            res = crosscheck_transformers(d)
        except ImportError as ex:  # pragma: no cover
            print("transformers unavailable, cross-check skipped:", ex)
            return
    res["note"] = ("independent float cross-check of the oracle's wiring vs HuggingFace transformers (fp32, tanh-GELU, eps 1e-5/1e-6 set to ggml's); "
                   "deviations are the oracle's deliberate ggml numerics: F16-rounded activations, fp16 LUTs, Q8 activation quantisation")
    (GOLD / "crosscheck.json").write_text(json.dumps(res, indent=1))
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
