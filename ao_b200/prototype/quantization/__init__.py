"""``ao_b200.prototype.quantization`` — the reference's prototype static float8 flow."""
from .float8_static_quant import PrototypeFloat8Tensor  # noqa: F401
from .quant_api import Float8StaticActivationFloat8WeightConfig  # noqa: F401
