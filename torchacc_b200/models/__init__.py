"""Native model definitions built on the sm_90a op set."""
from .llama import (LlamaConfig, LlamaDecoderLayer, LlamaForCausalLM, LlamaModel, ParallelContext, build_llama,
                    llama_config)
from .gpt2 import GPT2Config, GPT2Block, GPT2LMHeadModel, build_gpt2

__all__ = ["LlamaConfig", "LlamaDecoderLayer", "LlamaForCausalLM", "LlamaModel", "ParallelContext", "build_llama",
           "llama_config", "GPT2Config", "GPT2Block", "GPT2LMHeadModel", "build_gpt2"]
