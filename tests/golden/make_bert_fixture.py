"""Generates tests/golden/bert/hf_tiny/: a small Hugging Face BertModel and its fp64 outputs.

    config.json, model.safetensors   E 32, H 2 (head size 16), I 64, 2 layers, V 64, P 16,
                                     gelu_new (the encoder's tanh GELU), every parameter
                                     drawn at random (LayerNorm and biases included), fp32
    outputs.json                     fp64 `pooler_output` of the model (its fp32 weights
                                     widened to fp64, eager attention) on fixed rows of
                                     (input_ids, attention_mask, token_type_ids), padded
                                     rows included

The bert_lite files beside it are tf-models' TF2 BertEncoder test checkpoint
(extension/testdata of TensorFlow Ranking), copied unchanged.  This script needs
`transformers`, which no test imports.  Run from the repo root:
    python tests/golden/make_bert_fixture.py
"""
import json
import os

import torch
import transformers

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'bert', 'hf_tiny')
SEQ = 12


def rows():
  g = torch.Generator().manual_seed(7)
  lengths = [SEQ, 9, 5, 1]
  ids = torch.randint(1, 64, (len(lengths), SEQ), generator=g)
  ids[:, 0] = 2   # a [CLS]-like first token
  mask = torch.zeros(len(lengths), SEQ, dtype=torch.int64)
  types = torch.zeros(len(lengths), SEQ, dtype=torch.int64)
  for r, n in enumerate(lengths):
    mask[r, :n] = 1
    types[r, n // 2:n] = 1
    ids[r, n:] = 0
  return ids, mask, types


def main():
  torch.manual_seed(1234)
  config = transformers.BertConfig(
      vocab_size=64, hidden_size=32, num_hidden_layers=2, num_attention_heads=2,
      intermediate_size=64, max_position_embeddings=16, type_vocab_size=2,
      hidden_act='gelu_new', hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1,
      layer_norm_eps=1e-12, attn_implementation='eager')
  model = transformers.BertModel(config)
  with torch.no_grad():
    for name, p in model.named_parameters():
      if 'LayerNorm.weight' in name:
        p.copy_(1.0 + 0.2 * torch.randn_like(p))
      elif name.endswith('bias'):
        p.copy_(0.1 * torch.randn_like(p))
      else:
        p.copy_(0.3 * torch.randn_like(p))
  os.makedirs(OUT, exist_ok=True)
  model.save_pretrained(OUT, safe_serialization=True)
  ids, mask, types = rows()
  m64 = model.double().eval()
  with torch.no_grad():
    pooled = m64(input_ids=ids, attention_mask=mask, token_type_ids=types).pooler_output
  with open(os.path.join(OUT, 'outputs.json'), 'w') as f:
    json.dump({'input_ids': ids.tolist(), 'attention_mask': mask.tolist(),
               'token_type_ids': types.tolist(),
               'pooler_output': [[float(x) for x in r] for r in pooled.tolist()]}, f)
    f.write('\n')
  print('wrote', OUT)


if __name__ == '__main__':
  main()
