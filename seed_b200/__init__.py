"""seed_b200 -- Hopper (H100, sm_90a) implementation of the SEED visual-tokenizer encode path and the
llama_xformer forward path behind a C ABI (include/seedb200.h).  See README.md."""
__version__ = "0.1.0"
