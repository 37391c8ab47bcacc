"""virtex_b200 -- H100-native (sm_90a) implementation of the VirTex bicaptioning pretraining step."""
__version__ = "0.1.0"
