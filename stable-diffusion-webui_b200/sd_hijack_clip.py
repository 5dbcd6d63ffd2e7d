"""Text conditioning (SURVEY §8(f) row N4): the webui's prompt -> conditioning-tensor path with the CLIP text transformer
running on the sdxe engine. Host mirror of modules/sd_hijack_clip.py (same class / method names and argument meaning):

  PromptChunk, TextConditionalModel                 :9-285   75-token chunks, BREAK, comma backtracking, emphasis
    .tokenize_line / .process_texts / .forward / .process_tokens / .empty_chunk / .get_target_prompt_token_count
  FrozenCLIPEmbedderWithCustomWords                 :311-368 CLIP-L for SD1.x: encode_with_transformers incl.
                                                             CLIP_stop_at_last_layers ("clip skip")
  FrozenCLIPEmbedderForSDXLWithCustomWords          :371-384 CLIP-L inside SDXL: hidden_states[layer_idx], no final norm
  emphasis options                                   modules/sd_emphasis.py:24-70 (None / Ignore / Original / No norm)

`encode_with_transformers` = `sdxe_clip_forward` (engine kind SDXE_MODEL_CLIP_TEXT): embeddings, causal self-attention,
quick-GELU MLP, LayerNorms folded into the wgmma GEMMs. The tokenizer (BPE vocabulary files) is injected by the caller —
any object with the Hugging Face tokenizer surface the reference uses (`__call__(texts, truncation=False,
add_special_tokens=False)["input_ids"]`, `get_vocab()`, `bos_token_id`, `eos_token_id`). Textual-inversion embeddings
("custom words", :162-176, 219; modules/sd_hijack.py:340-366): every wrapper owns an `embedding_db`
(textual_inversion.EmbeddingDatabase); a prompt that names a registered embedding reserves its vectors' positions and the
engine overwrites those rows of the token embedding (`sdxe_clip_forward_fixes`).
"""
from __future__ import annotations

import math
from typing import List, Optional

import torch

from . import lib as L
from . import prompt_parser
from .engine import CLIPTextEngine, CLIPTextSpec
from .textual_inversion import EmbeddingDatabase


class PromptChunk:
    """token ids and multipliers of one 77-token chunk (start + 75 + end)."""

    def __init__(self):
        self.tokens: List[int] = []
        self.multipliers: List[float] = []
        self.fixes: list = []  # [(offset inside the 75 content tokens, Embedding)]: vectors go to positions offset + 1 ...


class TextOptions:
    """the `shared.opts` fields this path reads (defaults of modules/shared_options.py)."""

    emphasis = "Original"
    comma_padding_backtrack = 20
    CLIP_stop_at_last_layers = 1
    sdxl_clip_l_skip = False


# ---- modules/sd_emphasis.py ------------------------------------------------------------------------------------------
def _emphasis_none(z, multipliers):
    return z


def _emphasis_original(z, multipliers):
    original_mean = z.mean()
    z = z * multipliers.reshape(multipliers.shape + (1,)).expand(z.shape)
    return z * (original_mean / z.mean())  # "restoring original mean is likely not correct, but it seems to work well"


def _emphasis_no_norm(z, multipliers):
    return z * multipliers.reshape(multipliers.shape + (1,)).expand(z.shape)


EMPHASIS = {"None": _emphasis_none, "Ignore": _emphasis_none, "Original": _emphasis_original, "No norm": _emphasis_no_norm}


class TextConditionalModel:
    def __init__(self, opts: Optional[TextOptions] = None):
        self.opts = opts or TextOptions()
        self.chunk_length = 75
        self.return_pooled = False
        self.comma_token = None
        self.id_start = None
        self.id_end = None
        self.id_pad = None
        self.embedding_db = EmbeddingDatabase()    # the reference's model_hijack.embedding_db
        self.textual_inversion_key = "clip_l"      # which part of an SDXL embedding this encoder takes

    def empty_chunk(self) -> PromptChunk:
        chunk = PromptChunk()
        chunk.tokens = [self.id_start] + [self.id_end] * (self.chunk_length + 1)
        chunk.multipliers = [1.0] * (self.chunk_length + 2)
        return chunk

    def get_target_prompt_token_count(self, token_count: int) -> int:
        return math.ceil(max(token_count, 1) / self.chunk_length) * self.chunk_length

    def tokenize(self, texts):
        raise NotImplementedError

    def encode_with_transformers(self, tokens, fixes=None):
        raise NotImplementedError

    def fix_rows(self, batch_fixes, T: int):
        """EmbeddingsWithFixes.forward (modules/sd_hijack.py:347-366) as a list of row replacements: for batch row b and fix
        (offset, embedding), token positions offset + 1 ... take the embedding's vectors (as many as fit before position T),
        in order — a later fix overwrites an earlier one. -> [(b * T + position, vector [dim]), ...]"""
        out = []
        for b, fixes in enumerate(batch_fixes or []):
            for offset, embedding in fixes:
                vec = embedding.vec[self.textual_inversion_key] if isinstance(embedding.vec, dict) else embedding.vec
                emb_len = min(T - offset - 1, vec.shape[0])
                for j in range(emb_len):
                    out.append((b * T + offset + 1 + j, vec[j]))
        return out

    def tokenize_line(self, line: str):
        """one prompt -> (list of PromptChunk, token count). Emphasis syntax gives per-token multipliers; the word BREAK
        closes a chunk; a chunk that fills up within `comma_padding_backtrack` tokens after a comma is cut at that comma."""
        if self.opts.emphasis != "None":
            parsed = prompt_parser.parse_prompt_attention(line)
        else:
            parsed = [[line, 1.0]]
        tokenized = self.tokenize([text for text, _ in parsed])
        chunks: List[PromptChunk] = []
        cur = PromptChunk()
        token_count = 0
        last_comma = -1

        def close(is_last=False):
            nonlocal cur, token_count, last_comma
            token_count += len(cur.tokens) if is_last else self.chunk_length
            fill = self.chunk_length - len(cur.tokens)
            if fill > 0:
                cur.tokens += [self.id_end] * fill
                cur.multipliers += [1.0] * fill
            cur.tokens = [self.id_start] + cur.tokens + [self.id_end]
            cur.multipliers = [1.0] + cur.multipliers + [1.0]
            last_comma = -1
            chunks.append(cur)
            cur = PromptChunk()

        backtrack = self.opts.comma_padding_backtrack
        for tokens, (text, weight) in zip(tokenized, parsed):
            if text == "BREAK" and weight == -1:
                close()
                continue
            position = 0
            while position < len(tokens):
                token = tokens[position]
                if token == self.comma_token:
                    last_comma = len(cur.tokens)
                elif backtrack != 0 and len(cur.tokens) == self.chunk_length and last_comma != -1 and len(cur.tokens) - last_comma <= backtrack:
                    cut = last_comma + 1
                    moved_t, moved_m = cur.tokens[cut:], cur.multipliers[cut:]
                    cur.tokens, cur.multipliers = cur.tokens[:cut], cur.multipliers[:cut]
                    close()
                    cur.tokens, cur.multipliers = moved_t, moved_m
                if len(cur.tokens) == self.chunk_length:
                    close()
                embedding, name_tokens = self.embedding_db.find_embedding_at_position(tokens, position)
                if embedding is None:
                    cur.tokens.append(token)
                    cur.multipliers.append(weight)
                    position += 1
                    continue
                emb_len = int(embedding.vectors)           # :166-176: the vectors never straddle a chunk boundary
                if len(cur.tokens) + emb_len > self.chunk_length:
                    close()
                cur.fixes.append((len(cur.tokens), embedding))
                cur.tokens += [0] * emb_len
                cur.multipliers += [weight] * emb_len
                position += name_tokens
        if cur.tokens or not chunks:
            close(is_last=True)
        return chunks, token_count

    def process_texts(self, texts):
        token_count = 0
        cache = {}
        batch_chunks = []
        for line in texts:
            if line not in cache:
                cache[line], n = self.tokenize_line(line)
                token_count = max(n, token_count)
            batch_chunks.append(cache[line])
        return batch_chunks, token_count

    def forward(self, texts):
        """list of prompts -> [B, 77 * chunks, C] (and the pooled vector of the first chunk when return_pooled)."""
        batch_chunks, _ = self.process_texts(texts)
        chunk_count = max(len(x) for x in batch_chunks)
        zs, pooled0 = [], None
        for i in range(chunk_count):
            batch_chunk = [chunks[i] if i < len(chunks) else self.empty_chunk() for chunks in batch_chunks]
            z, pooled = self.process_tokens([x.tokens for x in batch_chunk], [x.multipliers for x in batch_chunk], [x.fixes for x in batch_chunk])
            zs.append(z)
            if i == 0:
                pooled0 = pooled
        out = torch.hstack(zs)
        return (out, pooled0) if self.return_pooled else out

    __call__ = forward

    def process_tokens(self, remade_batch_tokens, batch_multipliers, batch_fixes=None):
        tokens = torch.asarray(remade_batch_tokens)
        if self.id_end != self.id_pad:  # SD2-style tokenizers pad with a different id than end-of-text
            for pos in range(len(remade_batch_tokens)):
                index = remade_batch_tokens[pos].index(self.id_end)
                tokens[pos, index + 1:tokens.shape[1]] = self.id_pad
        if batch_fixes is not None and any(batch_fixes):
            z = self.encode_with_transformers(tokens, batch_fixes)
        else:
            z = self.encode_with_transformers(tokens)
        pooled = getattr(z, "pooled", None)
        fn = EMPHASIS.get(self.opts.emphasis, _emphasis_original)
        z = fn(z, torch.asarray(batch_multipliers).to(z.device, z.dtype))
        return z, pooled


class FrozenCLIPEmbedderWithCustomWords(TextConditionalModel):
    """CLIP-L text encoder of SD1.x on the sdxe engine. `state_dict` holds the `cond_stage_model.transformer.*` tensors
    (Hugging Face CLIPTextModel names, prefix stripped)."""

    def __init__(self, state_dict, tokenizer, spec: Optional[CLIPTextSpec] = None, dtype=torch.float16, device="cuda:0",
                 opts: Optional[TextOptions] = None):
        super().__init__(opts)
        self.tokenizer = tokenizer
        self.spec = spec or CLIPTextSpec.from_state_dict(state_dict)
        self.engine = CLIPTextEngine(self.spec, dtype=dtype, device=device)
        self.engine.load_state_dict(state_dict)
        self.engine.finalize()
        vocab = tokenizer.get_vocab()
        self.comma_token = vocab.get(",</w>", None)
        self.id_start = tokenizer.bos_token_id
        self.id_end = tokenizer.eos_token_id
        self.id_pad = self.id_end

    def tokenize(self, texts):
        return self.tokenizer(texts, truncation=False, add_special_tokens=False)["input_ids"]

    def encode_with_transformers(self, tokens, fixes=None):
        skip = int(self.opts.CLIP_stop_at_last_layers)
        # last_hidden_state == final_layer_norm(hidden_states[-1]); clip skip n: final_layer_norm(hidden_states[-n])
        return self.engine.forward(tokens, layer=self.spec.num_layers - (skip - 1 if skip > 1 else 0), final_norm=True,
                                   fixes=self.fix_rows(fixes, tokens.shape[1]))

    def load_embedding(self, path: str):
        """registers the embedding file under its base name if its width fits this encoder (textual_inversion.py:157-203)."""
        return self.embedding_db.load_from_file(path, self.tokenize, expected_shape=self.spec.hidden_size)

    def close(self):
        self.engine.close()


class FrozenCLIPEmbedderForSDXLWithCustomWords(FrozenCLIPEmbedderWithCustomWords):
    """CLIP-L as SDXL wires it (sgm FrozenCLIPEmbedder(layer="hidden", layer_idx=11)): a hidden state WITHOUT the final norm."""

    def __init__(self, *args, layer: str = "hidden", layer_idx: int = 11, **kwargs):
        super().__init__(*args, **kwargs)
        self.layer, self.layer_idx = layer, layer_idx

    def encode_with_transformers(self, tokens, fixes=None):
        n = self.spec.num_layers
        rows = self.fix_rows(fixes, tokens.shape[1])
        if self.opts.sdxl_clip_l_skip is True:
            idx = n + 1 - int(self.opts.CLIP_stop_at_last_layers)   # hidden_states[-skip] of n + 1 states
            return self.engine.forward(tokens, layer=idx, final_norm=False, fixes=rows)
        if self.layer == "last":
            return self.engine.forward(tokens, layer=n, final_norm=True, fixes=rows)
        idx = self.layer_idx if self.layer_idx >= 0 else n + 1 + self.layer_idx
        return self.engine.forward(tokens, layer=idx, final_norm=False, fixes=rows)


def open_clip_to_hf_state_dict(sd, prefix: str = "model."):
    """open_clip text-tower names (`FrozenOpenCLIPEmbedder2.model.*`: token_embedding, positional_embedding,
    transformer.resblocks.N.{ln_1, attn.in_proj_*, attn.out_proj, ln_2, mlp.c_fc, mlp.c_proj}, ln_final) -> the Hugging
    Face names the engine ingests. The fused in_proj is split into q / k / v."""
    out = {}
    g = lambda k: sd[prefix + k]  # noqa: E731
    out["text_model.embeddings.token_embedding.weight"] = g("token_embedding.weight")
    out["text_model.embeddings.position_embedding.weight"] = g("positional_embedding")
    n = 0
    while prefix + f"transformer.resblocks.{n}.ln_1.weight" in sd:
        s, d = f"transformer.resblocks.{n}.", f"text_model.encoder.layers.{n}."
        w, b = g(s + "attn.in_proj_weight"), g(s + "attn.in_proj_bias")
        c = w.shape[1]
        for i, name in enumerate(("q_proj", "k_proj", "v_proj")):
            out[d + f"self_attn.{name}.weight"] = w[i * c:(i + 1) * c]
            out[d + f"self_attn.{name}.bias"] = b[i * c:(i + 1) * c]
        for a, bname in (("attn.out_proj", "self_attn.out_proj"), ("ln_1", "layer_norm1"), ("ln_2", "layer_norm2"), ("mlp.c_fc", "mlp.fc1"),
                         ("mlp.c_proj", "mlp.fc2")):
            out[d + bname + ".weight"] = g(s + a + ".weight")
            out[d + bname + ".bias"] = g(s + a + ".bias")
        n += 1
    out["text_model.final_layer_norm.weight"] = g("ln_final.weight")
    out["text_model.final_layer_norm.bias"] = g("ln_final.bias")
    if n == 0:
        raise L.SdxeError("no open_clip text tower under prefix " + repr(prefix))
    return out


class FrozenOpenCLIPEmbedder2WithCustomWords(TextConditionalModel):
    """SDXL's second text encoder (sgm FrozenOpenCLIPEmbedder2: OpenCLIP ViT-bigG text tower, layer="penultimate",
    always_return_pooled) behind modules/sd_hijack_open_clip.py:38-71: z = the hidden state BEFORE the last block (no
    ln_final), z.pooled = ln_final(last hidden state)[end-of-text position] @ text_projection.
    `state_dict`: `conditioner.embedders.1.model.*` (open_clip names). The open_clip BPE tokenizer is injected
    (`encode(text) -> ids`, `encoder` dict); pad id is 0, not end-of-text (:45)."""

    def __init__(self, state_dict, tokenizer, num_heads: int = 20, dtype=torch.float16, device="cuda:0", opts: Optional[TextOptions] = None,
                 prefix: str = "model.", layer: str = "penultimate"):
        super().__init__(opts)
        self.tokenizer = tokenizer
        hf = open_clip_to_hf_state_dict(state_dict, prefix)
        self.spec = CLIPTextSpec.from_state_dict(hf, num_heads=num_heads, act="gelu")
        self.engine = CLIPTextEngine(self.spec, dtype=dtype, device=device)
        self.engine.load_state_dict(hf)
        self.engine.finalize()
        proj = state_dict[prefix + "text_projection"]                    # [width, embed_dim], used as x @ proj
        self.text_projection_t = proj.t().contiguous().to(device=device, dtype=dtype)  # [embed_dim, width] for out = A W^T
        self.layer = layer
        self.return_pooled = True
        self.comma_token = tokenizer.encoder.get(",</w>")
        self.id_start = tokenizer.encoder["<start_of_text>"]
        self.id_end = tokenizer.encoder["<end_of_text>"]
        self.id_pad = 0
        self.textual_inversion_key = "clip_g"      # modules/sd_hijack.py:62 wraps this tower's token embedding with 'clip_g'

    def tokenize(self, texts):
        return [self.tokenizer.encode(text) for text in texts]

    def encode_with_transformers(self, tokens, fixes=None):
        from . import ops

        n = self.spec.num_layers
        rows_fix = self.fix_rows(fixes, tokens.shape[1])
        z = self.engine.forward(tokens, layer=n - 1 if self.layer == "penultimate" else n, final_norm=self.layer != "penultimate", fixes=rows_fix)
        last = z if self.layer != "penultimate" else self.engine.forward(tokens, layer=n, final_norm=True, fixes=rows_fix)
        eot = tokens.to(last.device).argmax(dim=-1)                      # open_clip pools at the highest token id = <end_of_text>
        rows = last[torch.arange(last.shape[0], device=last.device), eot].contiguous()
        pooled = ops.gemm(rows, self.text_projection_t)                  # wgmma GEMM, M = number of prompts
        z.pooled = pooled  # the reference attaches the attribute to the hidden-state tensor (sd_hijack_open_clip.py:60-64)
        return z

    def close(self):
        self.engine.close()


def sdxl_size_embedding(values: torch.Tensor, dim: int = 256) -> torch.Tensor:
    """sgm ConcatTimestepEmbedderND(outdim=256): every scalar of `values` [B, k] -> sinusoidal embedding (cos | sin, the
    timestep_embedding of modules/sd_hijack_unet.py:58-78), concatenated -> [B, k * dim]."""
    half = dim // 2
    freqs = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float32, device=values.device) / half)
    args = values.reshape(-1)[:, None].float() * freqs[None]
    emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    return emb.reshape(values.shape[0], -1)


def sdxl_get_learned_conditioning(clip_l, clip_g, texts, width=1024, height=1024, crop_top=0, crop_left=0, is_negative_prompt=False):
    """modules/sd_models_xl.py:12-34 + sgm GeneralConditioner for SDXL-base: crossattn = CLIP-L hidden[11] | bigG penultimate
    (768 + 1280), vector = pooled (1280) | original size | crop | target size (3 x 2 x 256) = 2816. An all-empty negative
    prompt is zeroed (force_zero_embeddings=['txt'])."""
    zl = clip_l(texts)
    zg, pooled = clip_g(texts)
    if is_negative_prompt and all(x == "" for x in texts):
        zl, zg, pooled = torch.zeros_like(zl), torch.zeros_like(zg), torch.zeros_like(pooled)
    dev, B = zl.device, len(texts)
    size = torch.tensor([[height, width]], device=dev).repeat(B, 1)
    crop = torch.tensor([[crop_top, crop_left]], device=dev).repeat(B, 1)
    vec = torch.cat([pooled.float(), sdxl_size_embedding(size), sdxl_size_embedding(crop), sdxl_size_embedding(size)], dim=1)
    return {"crossattn": torch.cat([zl, zg.to(zl.dtype)], dim=-1), "vector": vec.to(zl.dtype)}
