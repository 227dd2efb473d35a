"""Metrics of the paper's experiments (reference `metrics/`): the edit distances of §5.1."""
