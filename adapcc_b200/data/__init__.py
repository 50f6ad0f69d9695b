"""Input pipeline of the conversational GPT-2 workload: tokenizer, PersonaChat-format data, pinned prefetch."""
from .personachat import (MODEL_INPUTS, DialogDataset, build_input_from_segments, build_tensors, corpus_of,  # noqa: F401
                          get_data_loaders, get_dataset, synthetic_personachat)
from .prefetch import PinnedPrefetcher, micro_batch_groups  # noqa: F401
from .tokenizer import SPECIAL_TOKENS, DialogTokenizer  # noqa: F401
