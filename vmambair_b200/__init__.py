"""vmambair_b200 -- H100-native Omni-Selective-Scan operator stack (drop-in for VmambaIR's OSS path)."""
__version__ = "0.1"
