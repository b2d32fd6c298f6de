"""The kernels at the shapes of the larger reference models (SURVEY.md Appendix A/B): one decoder layer of
Llama-3.1-8B / 70B / 405B geometry (GQA 4:1 / 8:1 / 16:1, hidden up to 16384, vocab 128256) trains on one GPU."""
import gc
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("model", ["meta-llama/Llama-3.1-8B", "meta-llama/Llama-3.1-70B", "meta-llama/Llama-3.1-405B"])
def test_one_layer_of_large_models_trains(model):
    from distributed_training_guide_b200.engine import TrainEngine

    eng = TrainEngine.create(model, parallelism="single", batch_size=1, seq_length=1024, lr=2e-4, num_layers=1)
    cfg = eng.config
    batch = eng.synthetic_batch(seed=0)
    losses = [float(eng.step(batch)) for _ in range(4)]
    eng.close()
    assert all(math.isfinite(l) for l in losses), losses
    # random init (std 0.02): logits have variance 0.02^2 * H, so the loss starts near ln(V) + var / 2
    expected = math.log(cfg.vocab_size) + 0.5 * 0.02 ** 2 * cfg.hidden_size
    assert abs(losses[0] - expected) < 1.0, (losses, expected)
    assert losses[-1] < losses[0] - 0.5, losses                     # and one batch is quickly memorised
    del eng
    gc.collect()                # engines hold reference cycles: free their buffers before the next (larger) case
    torch.cuda.empty_cache()
