"""MACE on the sm_90a engine (ScaleShiftMACE with scalar hidden features)."""
from .mace import MACECalculator_Dist
from .models import ScaleShiftMACE_Dist

__all__ = ["MACECalculator_Dist", "ScaleShiftMACE_Dist"]
