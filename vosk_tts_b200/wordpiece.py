"""The BERT WordPiece tokenizer that vosk_tts/model.py:60 loads: `BertWordPieceTokenizer(vocab, unk_token="[UNK]",
lowercase=True)` of Hugging Face's `tokenizers`, restated in Python so that a model directory loads without that compiled
package (as onnx_weights.py reads graphs without `onnx`).

The pipeline is the library's BertNormalizer, BertPreTokenizer, WordPiece model and BERT post-processor:
- clean text: NUL, U+FFFD and control characters (categories Cc, Cf, Co and Cs, except tab, newline and carriage return)
  are removed, and every remaining whitespace character becomes a space; unassigned code points (Cn) are kept, as the
  library keeps them;
- a space either side of every CJK ideograph;
- accents stripped (NFD, then the non-spacing marks Mn dropped), then each character lowercased on its own: `ещё` reads as
  `еще`, `мой` as `мои`;
- split on whitespace, and every punctuation character (ASCII punctuation or a Unicode P* category) is a word of its own;
- greedy longest-match WordPiece with the `##` prefix; a word longer than 100 characters, or one the vocabulary cannot
  cover, is one `[UNK]`;
- `[CLS]` first and `[SEP]` last.

Character classes come from Python's `unicodedata`, and the library carries its own Unicode tables, of other versions.  With
Python 3.12 (Unicode 15.0) and `tokenizers` 0.22, about 620 of the 1.1 million code points are classed differently: marks,
format characters and punctuation added to Unicode after the library's category tables (Newa, Sharada, Kawi, the
supplemental punctuation U+2E43 .. U+2E5D, ...), which the library treats as letters, and a few dozen letters whose
lowercase Unicode 16 added.  None is Cyrillic, Latin, or the punctuation of Russian text.
"""
import unicodedata

# the library's table: its fifth range starts at U+2B920 (BERT's original has U+2B820), so U+2B820 .. U+2B91F are not spaced
_CJK = ((0x4E00, 0x9FFF), (0x3400, 0x4DBF), (0x20000, 0x2A6DF), (0x2A700, 0x2B73F), (0x2B740, 0x2B81F), (0x2B920, 0x2CEAF),
        (0xF900, 0xFAFF), (0x2F800, 0x2FA1F))
# Unicode's White_Space property (what the library tests), not str.isspace, which also counts U+001C .. U+001F
_WHITESPACE = frozenset("\t\n\x0b\x0c\r \x85\xa0\u1680" + "".join(map(chr, range(0x2000, 0x200B))) + "\u2028\u2029\u202f\u205f\u3000")


def _is_control(ch):
    return ch not in "\t\n\r" and unicodedata.category(ch) in ("Cc", "Cf", "Co", "Cs")


def _is_punctuation(ch):
    o = ord(ch)
    return 33 <= o <= 47 or 58 <= o <= 64 or 91 <= o <= 96 or 123 <= o <= 126 or unicodedata.category(ch).startswith("P")


def _is_cjk(ch):
    o = ord(ch)
    return any(lo <= o <= hi for lo, hi in _CJK)


class Encoding:
    """The fields of a `tokenizers.Encoding` that vosk_tts/synth.py:26-41 reads."""

    def __init__(self, tokens, ids):
        self.tokens = tokens
        self.ids = ids
        self.attention_mask = [1] * len(ids)
        self.type_ids = [0] * len(ids)

    def __len__(self):
        return len(self.ids)


class BertWordPieceTokenizer:
    def __init__(self, vocab, unk_token="[UNK]", lowercase=True, max_input_chars_per_word=100):
        """vocab: a vocab.txt path (one token per line, its id the line number) or a dict token -> id."""
        if isinstance(vocab, dict):
            self.vocab = dict(vocab)
        else:
            self.vocab = {}
            with open(vocab, encoding="utf-8") as f:
                lines = f.read().split("\n")
            if lines and lines[-1] == "":
                lines.pop()
            for i, line in enumerate(lines):
                self.vocab[line.rstrip()] = i
        if not lowercase:
            raise ValueError("only the lowercasing tokenizer of vosk-tts models is implemented")
        for t in (unk_token, "[CLS]", "[SEP]"):
            if t not in self.vocab:
                raise ValueError("the vocabulary has no %s token" % t)
        self.unk_token = unk_token
        self.max_chars = int(max_input_chars_per_word)

    def normalize(self, text):
        out = []
        for ch in text:
            if ch == "\0" or ch == "\ufffd" or _is_control(ch):
                continue
            ch = " " if ch in _WHITESPACE else ch
            out.append(" %s " % ch if _is_cjk(ch) else ch)
        text = "".join(ch for ch in unicodedata.normalize("NFD", "".join(out)) if unicodedata.category(ch) != "Mn")
        return "".join(ch.lower() for ch in text)

    def pre_tokenize(self, text):
        words, cur = [], []
        for ch in text:
            if ch in _WHITESPACE or _is_punctuation(ch):
                if cur:
                    words.append("".join(cur))
                    cur = []
                if ch not in _WHITESPACE:
                    words.append(ch)
            else:
                cur.append(ch)
        if cur:
            words.append("".join(cur))
        return words

    def wordpiece(self, word):
        if len(word) > self.max_chars:
            return [self.unk_token]
        pieces, start = [], 0
        while start < len(word):
            end = len(word)
            while end > start:
                sub = word[start:end] if start == 0 else "##" + word[start:end]
                if sub in self.vocab:
                    break
                end -= 1
            if end == start:
                return [self.unk_token]
            pieces.append(sub)
            start = end
        return pieces

    def encode(self, text):
        tokens = ["[CLS]"] + [p for w in self.pre_tokenize(self.normalize(text)) for p in self.wordpiece(w)] + ["[SEP]"]
        return Encoding(tokens, [self.vocab[t] for t in tokens])
