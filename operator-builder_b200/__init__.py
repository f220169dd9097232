"""operator-builder_b200 -- H100-native marker scanning for operator-builder's `create api` hot path.

Only what the path needs: csrc/ (sm_90a CUDA kernels + the C ABI, built into libobmarkers.so),
lexer.py (host mirror of internal/markers/lexer's NewLexer/Run/NextLexeme over GPU tuples),
go/ (the cgo shim a Go build would compile).  Import as `operator_builder_b200` (the hyphenated
directory name is what the project brief prescribes; operator_builder_b200.py aliases it).
"""
from ._native import NativeError, SO_PATH  # noqa: F401
from .lexer import (BatchResult, Lexeme, LexemeType, Lexer, Position, Scanner, ZERO_LEXEME,  # noqa: F401
                    decode_doc_raw, generate_corpus_host, Registry, parse_doc_raw, Comm)
