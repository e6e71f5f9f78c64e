"""evo_b200: H100-native StripedHyena forward engine behind the evo-design/evo surface
(reference evo/__init__.py:3-6 exports Evo, generate, score_sequences, positional_entropies)."""
__version__ = "0.1.0"

from .models import Evo, load_checkpoint
from .generation import generate, Generator
from .scoring import score_sequences, positional_entropies, prepare_batch, logits_to_logprobs
from .tokenizer import CharLevelTokenizer
from .variants import score_variants, saturation_variants, apply_mutations
from .embeddings import embed_sequences
from .constraints import Constraints

__all__ = ["Evo", "load_checkpoint", "generate", "Generator", "score_sequences", "positional_entropies",
           "prepare_batch", "logits_to_logprobs", "CharLevelTokenizer", "score_variants", "saturation_variants", "apply_mutations",
           "embed_sequences", "Constraints"]
