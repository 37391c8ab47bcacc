from virtex_b200.metrics import CocoCaptionsEvaluator, TopkAccuracy, cider  # noqa: F401
