"""Drop-in for reference models/transformer.py (MakeAScene token transformer, tier 2) on the sm_90a kernels.

Same class names, constructor signatures, attribute names and state_dict keys (including the `transformer.mask`
buffer). Supported configuration = the reference's defaults: cogview_pb_relax=True (a softmax-invariant shift),
sandwich LayerNorm, no prescale, no rudalle_relax, dropout 0. The reference's `cache` / `use_cache` arguments raise
(its cache path is broken: transformer.py:73 vs :181, SURVEY.md 3.5); autoregressive sampling with a KV cache and
classifier-free guidance is `MakeAScene.generate` (new API, SURVEY.md 8f-3: specified by the non-cached forward).
Anything else raises — there is no fallback path.
"""
import math

import torch
import torch.nn as nn

from mas_b200 import ops


def gelu(x):
    """OpenAI tanh-GELU, transformer.py:11-14."""
    return ops.GeluFn.apply(x)


class LayerNorm(nn.LayerNorm):
    def forward(self, x, residual=None):
        return ops.LayerNormFn.apply(x, self.weight, self.bias, residual, self.eps)


class Linear(nn.Linear):
    def forward(self, x):
        return ops.LinearFn.apply(x, self.weight, self.bias)


class SelfAttention(nn.Module):
    def __init__(self, hidden_dim, num_attn_heads, attn_dropout_prob, out_dropout_prob, cogview_pb_relax=True, rudalle_relax=False):
        super().__init__()
        self.hidden_dim = hidden_dim
        self.num_attn_heads = num_attn_heads
        self.d = math.sqrt(self.hidden_dim // self.num_attn_heads)
        self.qkv = Linear(hidden_dim, 3 * hidden_dim)
        self.attn_drop = nn.Dropout(attn_dropout_prob)
        self.out_proj = Linear(hidden_dim, hidden_dim)
        self.out_drop = nn.Dropout(out_dropout_prob)
        self.cogview_pb_relax = cogview_pb_relax
        self.rudalle_relax = rudalle_relax
        if rudalle_relax or attn_dropout_prob or out_dropout_prob:
            raise NotImplementedError("rudalle_relax / dropout>0 have no kernel (reference defaults are off)")

    def forward(self, x, mask=None, use_cache=False, cache=None):
        if use_cache or cache is not None:
            raise NotImplementedError("KV cache: the reference path is broken (transformer.py:73 vs :181); no kernel")
        ctx = ops.CausalAttentionFn.apply(self.qkv(x), self.num_attn_heads)
        return self.out_proj(ctx), None


class MLP(nn.Module):
    def __init__(self, hidden_dim, dropout_prob, rudalle_relax=False):
        super().__init__()
        self.lin1 = Linear(hidden_dim, 4 * hidden_dim)
        self.lin2 = Linear(4 * hidden_dim, hidden_dim)
        self.dropout = nn.Dropout(dropout_prob)
        self.rudalle_relax = rudalle_relax
        if rudalle_relax or dropout_prob:
            raise NotImplementedError("rudalle_relax / dropout>0 have no kernel")

    def forward(self, x):
        return self.lin2(gelu(self.lin1(x)))


class TransformerLayer(nn.Module):
    def __init__(self, hidden_dim, num_attn_heads, attn_dropout_prop, out_dropout_prob, cogview_pb_relax=True,
                 cogview_sandwich_layernorm=True, cogview_layernorm_prescale=False, rudalle_relax=False):
        super().__init__()
        self.cogview_pb_relax = cogview_pb_relax
        self.cogview_sandwich_layernorm = cogview_sandwich_layernorm
        self.cogview_layernorm_prescale = cogview_layernorm_prescale
        self.rudalle_relax = rudalle_relax
        if cogview_layernorm_prescale or rudalle_relax:
            raise NotImplementedError("layernorm prescale / rudalle_relax have no kernel")
        self.ln_in = LayerNorm(hidden_dim, eps=1e-5)
        self.ln_out = LayerNorm(hidden_dim, eps=1e-5)
        if cogview_sandwich_layernorm:
            self.first_ln_sandwich = LayerNorm(hidden_dim, eps=1e-5)
            self.second_ln_sandwich = LayerNorm(hidden_dim, eps=1e-5)
        self.attn = SelfAttention(hidden_dim=hidden_dim, num_attn_heads=num_attn_heads, attn_dropout_prob=attn_dropout_prop,
                                  out_dropout_prob=out_dropout_prob, cogview_pb_relax=cogview_pb_relax, rudalle_relax=rudalle_relax)
        self.mlp = MLP(hidden_dim=hidden_dim, dropout_prob=out_dropout_prob, rudalle_relax=rudalle_relax)

    def forward(self, x, mask=None, cache=None, use_cache=False, mlp_cache=False):
        if use_cache or cache is not None:
            raise NotImplementedError("KV cache has no kernel")
        attn_out, _ = self.attn(self.ln_in(x))
        if self.cogview_sandwich_layernorm:
            x = self.first_ln_sandwich(attn_out, residual=x)      # x + LN(attn_out), fused
        else:
            x = x + attn_out
        mlp_out = self.mlp(self.ln_out(x))
        if self.cogview_sandwich_layernorm:
            x = self.second_ln_sandwich(mlp_out, residual=x)
        else:
            x = x + mlp_out
        return x, None


class Transformer(nn.Module):
    def __init__(self, num_layers, hidden_dim, num_attn_heads, image_tokens_per_dim, seg_tokens_per_dim, text_length,
                 attn_dropout_prop=0, out_dropout_prob=0, cogview_pb_relax=True, cogview_sandwich_layernorm=True,
                 cogview_layernorm_prescale=False, rudalle_relax=False):
        super().__init__()
        self.num_layers = num_layers
        self.cogview_pb_relax = cogview_pb_relax
        self.rudalle_relax = rudalle_relax
        self.layers = nn.ModuleList([
            TransformerLayer(hidden_dim, num_attn_heads, attn_dropout_prop, out_dropout_prob, cogview_pb_relax,
                             cogview_sandwich_layernorm, cogview_layernorm_prescale, rudalle_relax) for _ in range(num_layers)])
        self.register_buffer("mask", self._create_mask(text_length, seg_tokens_per_dim, image_tokens_per_dim))
        self.final_ln = LayerNorm(hidden_dim, eps=1e-5)

    def _create_mask(self, text_length, seg_tokens_per_dim, image_tokens_per_dim):
        size = text_length + seg_tokens_per_dim ** 2 + image_tokens_per_dim ** 2
        return torch.tril(torch.ones(size, size, dtype=torch.float32))

    def forward(self, x, attn_mask=None, cache=None, use_cache=None):
        # attn_mask * self.mask is plain causal for every mask MakeAScene builds (transformer.py:262-263, 366-370):
        # the kernels implement the causal mask directly.
        if use_cache or cache:
            raise NotImplementedError("KV cache has no kernel")
        if attn_mask is not None:
            S = x.shape[1]
            am = attn_mask.to(self.mask.device, self.mask.dtype)
            while am.dim() > 2:        # [B,1,S,S] / [1,1,S,S] -> [S,S] only if it is the same for every row
                if am.shape[0] != 1 and not bool((am == am[:1]).all()):
                    raise RuntimeError("per-sample attention masks have no kernel (only the causal mask is implemented)")
                am = am[0]
            eff = am[:S, :S] * self.mask[:S, :S]
            if not torch.equal(eff != 0, self.mask[:S, :S] != 0):
                raise RuntimeError("attn_mask * causal mask is not the plain causal mask: only causal attention has a kernel "
                                   "(a padding / prefix mask would silently be ignored otherwise)")
        for layer in self.layers:
            x, _ = layer(x)
        return self.final_ln(x), {}


def _param_version(model):
    return tuple((p._version, p.data_ptr()) for p in model.parameters())


class _GraphedDecoder:
    """KV caches + one captured CUDA graph per image position for MakeAScene.generate(use_graphs=True).

    A decode step is ~250 launches of a few microseconds each (24 layers x 10 kernels): launched from Python it is
    host-bound (~22 us per launch). The kernels only depend on the position through launch parameters, so each position
    gets its own graph (captured on first use, replayed in position order afterwards; the graphs share one memory pool).
    The caches are fp32 up to 8 rows and fp16 above (the cache read dominates a step at a few hundred rows).
    Above 8 rows the decode Linears read the fp16 weight images of ops.decode_weight_image: they are built here, before any
    capture, and held by the decoder, so the graphs never record a packing launch and never outlive the images they read.
    `version` records every parameter's version and storage: generate() builds a new decoder when it changes."""

    def __init__(self, model, rows, dev):
        layers = model.transformer.layers
        heads = layers[0].attn.num_attn_heads
        hd = model.hidden_dim // heads
        self.model, self.rows = model, rows
        dt = torch.float32 if rows <= ops.DECODE_F32_ROWS else torch.float16
        self.kc = [torch.empty((rows, heads, model.total_length, hd), dtype=dt, device=dev) for _ in layers]
        self.vc = [torch.empty_like(k) for k in self.kc]
        self.version = _param_version(model)
        self.images = []
        if rows > ops.DECODE_F32_ROWS:
            lins = [m for l in layers for m in (l.attn.qkv, l.attn.out_proj, l.mlp.lin1, l.mlp.lin2)] + [model.to_logits[1]]
            self.images = [ops.decode_weight_image(m.weight) for m in lins if m.weight.shape[1] % 64 == 0]
        self.tok = torch.zeros(rows, dtype=torch.long, device=dev)
        self.pool = torch.cuda.graph_pool_handle()
        self.graphs, self.keep = {}, {}

    def eager_step(self, t, tok_all, prefix):
        m = self.model
        dev, ip, R = tok_all.device, m.image_tokens_per_dim, self.rows
        row = torch.full((1,), t // ip, dtype=torch.long, device=dev)
        col = torch.full((1,), t % ip, dtype=torch.long, device=dev)
        return self._body(tok_all, row, col, prefix + t)

    def _body(self, tok, row, col, pos):
        m, R = self.model, self.rows
        emb = ops.EmbedFn.apply([(tok.view(R, 1), row, col, 0)], 1, m.hidden_dim, m.image_token_embedding.weight,
                                m.image_row_embeddings.weight, m.image_col_embeddings.weight)
        return m._logits_of(m._decode_step(emb.view(R, m.hidden_dim), self.kc, self.vc, pos), normed=True)

    def graphed_step(self, t, tok_all, prefix):
        self.tok.copy_(tok_all)
        if t not in self.graphs:
            dev, ip = tok_all.device, self.model.image_tokens_per_dim
            row = torch.full((1,), t // ip, dtype=torch.long, device=dev)
            col = torch.full((1,), t % ip, dtype=torch.long, device=dev)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, pool=self.pool):
                out = self._body(self.tok, row, col, prefix + t)
            self.graphs[t], self.keep[t] = g, (out, row, col)
        self.graphs[t].replay()
        return self.keep[t][0]


class MakeAScene(nn.Module):
    def __init__(self, num_layers, hidden_dim, num_attn_heads, image_vocab_size, seg_vocab_size, text_vocab_size,
                 image_tokens_per_dim, seg_tokens_per_dim, text_length):
        super().__init__()
        self.image_tokens_per_dim = image_tokens_per_dim
        self.seg_tokens_per_dim = seg_tokens_per_dim
        self.image_length = image_tokens_per_dim ** 2
        self.seg_length = seg_tokens_per_dim ** 2
        self.text_length = text_length
        self.total_length = self.text_length + self.seg_length + self.image_length
        self.text_vocab_size = text_vocab_size
        self.hidden_dim = hidden_dim
        self.transformer = Transformer(num_layers, hidden_dim, num_attn_heads, image_tokens_per_dim, seg_tokens_per_dim, text_length)
        self.image_token_embedding = nn.Embedding(image_vocab_size, hidden_dim)
        self.seg_token_embedding = nn.Embedding(seg_vocab_size, hidden_dim)
        self.text_token_embedding = nn.Embedding(text_vocab_size, hidden_dim)
        self.text_pos_embeddings = torch.nn.Embedding(text_length, hidden_dim)
        self.seg_row_embeddings = torch.nn.Embedding(seg_tokens_per_dim, hidden_dim)
        self.seg_col_embeddings = torch.nn.Embedding(seg_tokens_per_dim, hidden_dim)
        self.image_row_embeddings = torch.nn.Embedding(image_tokens_per_dim, hidden_dim)
        self.image_col_embeddings = torch.nn.Embedding(image_tokens_per_dim, hidden_dim)
        for m in (self.text_pos_embeddings, self.seg_row_embeddings, self.seg_col_embeddings, self.image_row_embeddings,
                  self.image_col_embeddings):
            self._init_weights(m)
        self.to_logits = torch.nn.Sequential(LayerNorm(hidden_dim), Linear(hidden_dim, image_vocab_size))

    def reset_sampler(self):
        """Drops the cached KV buffers / CUDA graphs of generate(use_graphs=True) (they are rebuilt by themselves when a
        parameter changes)."""
        self._sampler = None

    def _init_weights(self, module):
        if isinstance(module, (nn.Linear, nn.Embedding)):
            module.weight.data.normal_(mean=0.0, std=0.02)
            if isinstance(module, nn.Linear) and module.bias is not None:
                module.bias.data.zero_()
        elif isinstance(module, nn.LayerNorm):
            module.bias.data.zero_()
            module.weight.data.fill_(1.0)

    def _embed(self, text_tokens, seg_tokens, img_tokens):
        """Token + position embeddings of the concatenated sequence, transformer.py:350-364."""
        dev = text_tokens.device
        text_range = torch.arange(self.text_length, device=dev) + (self.text_vocab_size - self.text_length)
        text_tokens = torch.where(text_tokens == 0, text_range, text_tokens)      # pad-id trick, transformer.py:350-353
        ar = lambda n: torch.arange(n, dtype=torch.long, device=dev)
        sp, ip = self.seg_tokens_per_dim, self.image_tokens_per_dim
        segs = [(text_tokens, ar(text_tokens.shape[1]), None, 0),
                (seg_tokens, ar(seg_tokens.shape[1]) // sp, ar(seg_tokens.shape[1]) % sp, text_tokens.shape[1])]
        tables = [self.text_token_embedding.weight, self.text_pos_embeddings.weight, self.text_pos_embeddings.weight,
                  self.seg_token_embedding.weight, self.seg_row_embeddings.weight, self.seg_col_embeddings.weight]
        total = text_tokens.shape[1] + seg_tokens.shape[1]
        if img_tokens is not None:
            segs.append((img_tokens, ar(img_tokens.shape[1]) // ip, ar(img_tokens.shape[1]) % ip, total))
            tables += [self.image_token_embedding.weight, self.image_row_embeddings.weight, self.image_col_embeddings.weight]
            total += img_tokens.shape[1]
        return ops.EmbedFn.apply(segs, total, self.hidden_dim, *tables)

    def forward(self, text_tokens, seg_tokens, img_tokens):
        """Logits [B, image_length, V] predicting every image token from its prefix (transformer.py:366-378). The reference
        computes to_logits over all 640 positions and slices afterwards; LayerNorm and Linear act row by row, so slicing the
        hidden states first gives the same values (and the same, zero, gradient for the dropped rows) at 40 % of the work."""
        emb = self._embed(text_tokens, seg_tokens, img_tokens)
        out, _ = self.transformer(emb)
        out = out[:, -self.image_length - 1:-1, :].contiguous()
        return self.to_logits[1](self.to_logits[0](out))

    def loss(self, text_tokens, seg_tokens, img_tokens):
        """train.py:150-153 in one call: F.cross_entropy(forward(...).view(-1, V), img_tokens.view(-1)) on the fused
        cross-entropy kernels (mas_ce_forward / mas_ce_backward: no log-softmax tensor, the gradient is written once)."""
        return ops.cross_entropy(self.forward(text_tokens, seg_tokens, img_tokens), img_tokens)

    # ---- sampling (SURVEY.md 8f-3) ---------------------------------------------------------------------------
    def _prefill(self, emb, kc, vc):
        """Full causal pass over the text+segmentation prefix with the training kernels, recording every layer's k / v."""
        x = emb
        heads = self.transformer.layers[0].attn.num_attn_heads
        for li, layer in enumerate(self.transformer.layers):
            qkv = layer.attn.qkv(layer.ln_in(x))
            ops.kv_append(qkv, kc[li], vc[li], 0)
            a = layer.attn.out_proj(ops.CausalAttentionFn.apply(qkv, heads))
            x = layer.first_ln_sandwich(a, residual=x) if layer.cogview_sandwich_layernorm else x + a
            m = layer.mlp(layer.ln_out(x))
            x = layer.second_ln_sandwich(m, residual=x) if layer.cogview_sandwich_layernorm else x + m
        return x[:, -1].contiguous()

    def _decode_step(self, x, kc, vc, pos):
        """One new token per row (x [R,H], absolute position pos) through all layers against the cache; returns
        final_ln(hidden). Seven launches per layer: qkv, attention (+ cache append), out_proj, the sandwich LayerNorm chained
        with the next input LayerNorm (mas_layernorm2_forward), lin1 (+GELU), lin2, the second chained pair."""
        layers = self.transformer.layers
        if not all(l.cogview_sandwich_layernorm for l in layers) or x.shape[-1] % 4 or x.shape[-1] > 4096:
            return self.transformer.final_ln(self._decode_step_plain(x, kc, vc, pos))
        y = layers[0].ln_in(x)
        for li, layer in enumerate(layers):
            at, mlp = layer.attn, layer.mlp
            qkv = ops.linear_small(y, at.qkv.weight, at.qkv.bias)
            a = ops.linear_small(ops.attn_decode_append(qkv, kc[li], vc[li], pos), at.out_proj.weight, at.out_proj.bias)
            x, y = ops.layernorm2(a, layer.first_ln_sandwich, x, layer.ln_out)        # x + LN(a), then the MLP's input norm
            m = ops.linear_small(y, mlp.lin1.weight, mlp.lin1.bias, act=1)
            m = ops.linear_small(m, mlp.lin2.weight, mlp.lin2.bias)
            nxt = layers[li + 1].ln_in if li + 1 < len(layers) else self.transformer.final_ln
            x, y = ops.layernorm2(m, layer.second_ln_sandwich, x, nxt)
        return y

    def _decode_step_plain(self, x, kc, vc, pos):
        """The unfused form (configurations without the sandwich LayerNorm); returns the hidden state before final_ln."""
        for li, layer in enumerate(self.transformer.layers):
            at, mlp = layer.attn, layer.mlp
            qkv = ops.linear_small(layer.ln_in(x), at.qkv.weight, at.qkv.bias)
            ops.kv_append(qkv.view(qkv.shape[0], 1, -1), kc[li], vc[li], pos)
            a = ops.linear_small(ops.attn_decode(qkv, kc[li], vc[li], pos + 1), at.out_proj.weight, at.out_proj.bias)
            x = layer.first_ln_sandwich(a, residual=x) if layer.cogview_sandwich_layernorm else x + a
            m = ops.linear_small(layer.ln_out(x), mlp.lin1.weight, mlp.lin1.bias, act=1)
            m = ops.linear_small(m, mlp.lin2.weight, mlp.lin2.bias)
            x = layer.second_ln_sandwich(m, residual=x) if layer.cogview_sandwich_layernorm else x + m
        return x

    def _logits_of(self, hidden, normed=False):
        """to_logits on hidden states [R,H]; normed: final_ln has been applied already (decode steps)."""
        f = hidden if normed else self.transformer.final_ln(hidden)
        h = self.to_logits[0](f)
        return ops.linear_small(h, self.to_logits[1].weight, self.to_logits[1].bias)

    @torch.no_grad()
    def generate(self, text_tokens, seg_tokens, guidance_scale=None, uncond_text_tokens=None, temperature=1.0, top_k=None,
                 generator=None, img_tokens=None, return_logits=False, use_graphs=False, top_p=None, img_mask=None):
        """Autoregressive sampling of the image tokens with a KV cache; optional classifier-free guidance
        (logits = uncond + scale * (cond - uncond), the unconditional stream sees padded text; Make-A-Scene paper 3.4).

        text_tokens [B,text_length], seg_tokens [B,seg_length] int64. A call decodes R = B rows (2B with guidance); memory is
        the only limit on R. Up to 8 rows the decode steps are strict fp32 (weights and KV cache). More rows run the decode
        Linear layers on fp16 operands with fp32 accumulation and keep K / V in fp16 caches: the arithmetic of the model's own
        training forward. The prefix pass always runs the training kernels.
        The draw at each position, per row (ru-DALL-E's top_k_top_p_filtering chain, one kernel launch):
          z = logits / temperature; top_k keeps the k largest (ties with the k-th kept); top_p (None or >= 1: off, <= 0:
          ValueError) keeps, of those, every entry whose softmax mass of kept entries with a strictly larger z is <= top_p
          (equal values are kept or dropped together; the largest always stays); the token is the inverse CDF of softmax(z)
          over the kept set at a uniform, in index order. temperature 0 = greedy (the first index of the maximum).
        img_tokens (optional [B,image_length] int64) are fed instead of the sampled ones at every position (teacher forcing —
        what the parity test uses). With img_mask ([B,image_length] bool on the same device) only the positions where it is
        set are forced (image prompts: completion, outpainting, editing a region); the others are drawn, conditioned on all
        earlier tokens, forced or drawn. With guidance a forced token goes to both streams. When sampling with img_mask, the
        B uniforms are drawn at every position, forced or not, so a row's random stream does not depend on the mask: an
        all-false mask gives the tokens of the unprompted call with the same generator.
        Returns tokens [B,image_length] (and the per-position logits [B,image_length,V], mixed and unfiltered, when
        return_logits=True).
        use_graphs: replay each position's decode step from a CUDA graph (captured at first use and kept on the module for
        the same row count; captured again after any parameter changes, in place or by replaced storage)."""
        B = text_tokens.shape[0]
        dev = text_tokens.device
        if top_p is not None and not float(top_p) > 0:
            raise ValueError("top_p must be > 0 (None or >= 1: no nucleus filter), got %r" % (top_p,))
        if img_mask is not None:
            want = (B, self.image_length)
            if img_tokens is None:
                raise ValueError("img_mask selects positions of img_tokens: pass img_tokens too")
            if not isinstance(img_mask, torch.Tensor) or img_mask.dtype != torch.bool or tuple(img_mask.shape) != want:
                raise ValueError("img_mask must be a bool tensor of shape %s" % (want,))
            if img_tokens.dtype != torch.int64 or tuple(img_tokens.shape) != want:
                raise ValueError("img_tokens must be an int64 tensor of shape %s" % (want,))
            if img_mask.device != dev or img_tokens.device != dev:
                raise ValueError("img_tokens and img_mask must be on the device of text_tokens (%s)" % dev)
            img_tokens, img_mask = img_tokens.contiguous(), img_mask.contiguous()
        cfg = guidance_scale is not None and float(guidance_scale) != 1.0
        if cfg:
            if uncond_text_tokens is None:
                uncond_text_tokens = torch.zeros_like(text_tokens)          # all padding -> the per-position pad ids
            text_all = torch.cat([text_tokens, uncond_text_tokens], 0)
            seg_all = torch.cat([seg_tokens, seg_tokens], 0)
        else:
            text_all, seg_all = text_tokens, seg_tokens
        R = text_all.shape[0]
        dec = getattr(self, "_sampler", None)
        if dec is None or dec.rows != R or dec.tok.device != dev or not use_graphs or dec.version != _param_version(self):
            dec = _GraphedDecoder(self, R, dev)
            if use_graphs:
                self._sampler = dec
        kc, vc = dec.kc, dec.vc
        prefix = text_all.shape[1] + seg_all.shape[1]
        logits = self._logits_of(self._prefill(self._embed(text_all, seg_all, None), kc, vc))
        toks, kept = [], []
        for t in range(self.image_length):
            mixed = ops.cfg_mix(logits[:B], logits[B:], guidance_scale) if cfg else logits
            if return_logits:
                kept.append(mixed)
            prompt = (img_tokens[:, t], img_mask[:, t]) if img_mask is not None else None
            if img_tokens is not None and prompt is None:
                tok = img_tokens[:, t]
            elif not temperature and prompt is None:
                tok = mixed.argmax(-1)
            else:   # prompt, temperature, top-k / top-p filters, softmax and the draw in one kernel; torch only supplies the uniforms
                u = None
                if temperature:
                    if generator is not None and generator.device.type != dev.type:
                        u = torch.rand(B, generator=generator).to(dev)
                    else:
                        u = torch.rand(B, device=dev, generator=generator)
                tok = ops.sample_topk(mixed, float(temperature), top_k, u, top_p=top_p, prompt=prompt)
            toks.append(tok)
            if t == self.image_length - 1:
                break
            tok_all = torch.cat([tok, tok], 0) if cfg else tok
            logits = (dec.graphed_step if use_graphs else dec.eager_step)(t, tok_all, prefix)
        tokens = torch.stack(toks, 1)
        if return_logits:
            return tokens, torch.stack(kept, 1)
        return tokens
