"""Import-path alias: `import virtex...` resolves to the H100-native implementation in `virtex_b200` for the
bicaptioning pretraining path (same module layout as the reference for the parts of its surface that are in scope)."""
from virtex_b200 import __version__  # noqa: F401
