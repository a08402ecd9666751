"""``llama_sft.py`` with packed rows: several Alpaca samples per row of ``max_length`` tokens, attention and rotary
positions restarting at every sample (``PackedSFTDataset``), so the GEMMs and attention run on far fewer padding
tokens.  Everything else is the same recipe.  ``max_length`` is the row length; it may differ from the length the
corpus was prepared at (``prepare_alpaca.py --max-seq-length``), but no prepared sample may be longer (the dataset
raises) and it must not exceed ``cfg.max_position_embeddings``."""
import copy
import os

from libai_b200.config import LazyCall, OmegaConf
from libai_b200.data.build import build_nlp_train_loader
from projects.common.sft import PackedSFTDataset
from projects.Llama.configs import llama_sft
from projects.Llama.configs.llama_sft import cfg, dataset_path, graph, model, optim, tokenization, train  # noqa: F401

max_length = 512

# a config of its own: llama_sft's dataloader object is left as it is
dataloader = OmegaConf.create()
dataloader.train = LazyCall(build_nlp_train_loader)(
    dataset=[LazyCall(PackedSFTDataset)(path=os.path.join(dataset_path, "train"), max_length=max_length,
                                        tokenizer=tokenization.tokenizer)],
)
dataloader.test = copy.deepcopy(llama_sft.dataloader.test)
