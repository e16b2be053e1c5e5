"""H100-native data-parallel hot path for lartpang/Distributed-SOD-Project (see DESIGN.md)."""
__version__ = "0.1.0"
