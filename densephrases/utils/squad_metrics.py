from densephrases_b200.rc import compute_predictions_logits, squad_evaluate  # noqa: F401  (squad_metrics.py:221-254, 408-684; span decoding on the GPU)
