"""models.peft_model -- mirror of the reference's src/model/peft_model.py get_peft_model_with_resize_embedding for
inference with a trained LoRA checkpoint (seed_b200/peft.py).

Differences from the reference:
  * a `peft_config` (building a trainable adapter) raises NotImplementedError: only `model_id` is supported;
  * a DictConfig `model` is instantiated in fp16 whatever `torch_dtype` says, because seed_b200 runs LLaMA in fp16
    only and both eval scripts call `.half()` on the result next;
  * omegaconf / hydra are imported only when `model` is a config, so they are not dependencies otherwise.
"""
from seed_b200.peft import PeftModel


def get_peft_model_with_resize_embedding(model, peft_config=None, model_id=None, tokenizer=None, torch_dtype='bf16'):
    if peft_config is not None:
        raise NotImplementedError("peft_config (training a new adapter) is not supported; pass model_id")
    if model_id is None:
        raise ValueError("exactly one of peft_config and model_id must be given")
    if type(model).__name__ == "DictConfig":
        import hydra

        model = hydra.utils.instantiate(model, torch_dtype="fp16")
    if tokenizer is not None:
        print(f'Length of tokenizer and resize embedding: {len(tokenizer)}')
        model.resize_token_embeddings(len(tokenizer))
    return PeftModel.from_pretrained(model=model, model_id=model_id)
