"""tokenizers_b200 -- CUDA (H100) batched tokenization engine behind the `Tokenizer.encode_batch` surface of
huggingface/tokenizers (ByteLevel-BPE and Whitespace+WordPiece).  See DESIGN.md / INTEGRATION.md."""
from .tokenizer import Tokenizer, Encoding, BatchEncoding, UnsupportedConfig, parse_tokenizer_json  # noqa: F401
from ._lib import B2TError  # noqa: F401

__version__ = "0.1.0"
