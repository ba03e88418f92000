"""tensorflowonspark_b200: a Hopper-native framework with the capabilities and
public API of yahoo/TensorFlowOnSpark (reference: tensorflowonspark/__init__.py:1-5)."""
import logging

logging.basicConfig(level=logging.INFO,
                    format="%(asctime)s %(levelname)s (%(threadName)s-%(process)d) %(message)s")

__version__ = "0.2.0"
