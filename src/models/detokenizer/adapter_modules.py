"""`src.models.detokenizer.adapter_modules.{SDXLAdapter,SDXLAdapterWithLatentImage}` -> H100 engine
(reference: src/models/detokenizer/adapter_modules.py:11-287)."""
from seedx_b200.adapter import SDXLAdapter, SDXLAdapterWithLatentImage  # noqa: F401
