"""Test helper: a synthetic workspace the reference's run_pretrain_distributed_gpt3.py can run on - tiny model
directory (config.json / visual json / tokenizer.json), the task yaml with the reference's own keys
(configs/pretrain/gpt3_1.3B/pretrain_gpt3_freezeGPT_youku_v0.yaml), a csv in the loader's format
(dataset/video_pretrain_dataset.py:22-24) and .npy clips for the decord stand-in."""
import json
import os

import numpy as np

from oracle import port


def make_workspace(td, num_videos=8, batch_size=2, max_length=8, num_workers=0):
    from tokenizers import Tokenizer, models, pre_tokenizers
    md = os.path.join(td, "text_decoder")
    os.makedirs(md, exist_ok=True)
    vcfg = dict(port.VCFG_TINY, pretrained_ckpt=None, grad_ckpt=False, drop_path=0, stop_grad_conv1=False,
                use_shared_rel_pos_bias=False, use_abs_pos_emb=True)
    with open(os.path.join(td, "vis.json"), "w") as f:
        json.dump(vcfg, f)
    with open(os.path.join(md, "config.json"), "w") as f:
        json.dump(dict(port.GCFG_TINY, hidden_dropout=0.0, attention_dropout=0.0), f)
    vocab = {"<|endoftext|>": 0, "<sep>": 1, "[UNK]": 2, "\n": 3}
    words = "a b c d e f g hello world video cat dog runs on the grass".split()
    for i, w in enumerate(words):
        vocab[w] = 4 + i
    tok = Tokenizer(models.WordLevel(vocab, unk_token="[UNK]"))
    tok.pre_tokenizer = pre_tokenizers.Whitespace()
    tok.save(os.path.join(md, "tokenizer.json"))
    vids = os.path.join(td, "videos")
    os.makedirs(vids, exist_ok=True)
    rng = np.random.default_rng(0)
    rows = ["video_id:FILE,title"]
    for i in range(num_videos):
        np.save(os.path.join(vids, f"clip{i}.npy"), rng.integers(0, 256, (6, 40, 48, 3), dtype=np.uint8))
        rows.append(f"clip{i}.npy,{' '.join(rng.choice(words, 4))}")
    with open(os.path.join(td, "pretrain.csv"), "w") as f:
        f.write("\n".join(rows) + "\n")
    cfg = f"""train_file: [
  {os.path.join(td, 'pretrain.csv')}
]
read_local_data: true

train_video_root: "{vids}/"

text_decoder: '{md}/'
text_cfg: {os.path.join(md, 'config.json')}
visual_cfg: '{os.path.join(td, 'vis.json')}'

megatron_cfg: {{
  "world_size": 1,
  "model_parallel_size": 1,
  "tensor_model_parallel_size": 1,
}}

batch_size: {batch_size}
num_workers: {num_workers}
max_length: {max_length}

freeze_vit: false
freeze_text_decoder: true

num_learnable_token: 8
use_contrastive: false

temp: 0.07
embed_dim: 256

optimizer: {{
  lr: 1e-4,
  opt: "AdamW",
  weight_decay: 0.05,
  clip_grad: 3.0,
  opt_betas: [0.9, 0.999],
  opt_eps: 1e-6
}}

schedular: {{
  epochs: 1,
  min_lr: 1e-6,
  warmup_epochs: -1,
  warmup_steps: 1,
  lr_sched_type: "cosine"
}}
"""
    path = os.path.join(td, "pretrain_tiny.yaml")
    with open(path, "w") as f:
        f.write(cfg)
    return dict(config=path, model_dir=md, output_dir=os.path.join(td, "out"), videos=vids)
