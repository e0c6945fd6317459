"""Text -> token strings without spaCy: a restatement of spaCy 2.x's rule-based English tokenizer, the word splitter
behind fastai 1.0.53's ``Tokenizer(SpacyTokenizer('en'))`` that the reference's learner uses to numericalise issues
(Issue_Embeddings/flask_app/inference.py:51-53, :174-182; SURVEY.md section 8, row f-1 "next").

Boundary code, host only; the GPU path starts at token ids.  PARITY UNPINNED: spaCy is not installed in this image, so
the rules below are restated from the published spaCy 2.1 sources (``spacy/tokenizer.pyx`` -- the whitespace /
prefix / suffix / infix / special-case loop; ``spacy/lang/punctuation.py`` and ``char_classes.py`` -- the character
classes; ``spacy/lang/en/tokenizer_exceptions.py`` and ``lang/tokenizer_exceptions.py`` -- contractions,
abbreviations, emoticons) and checked only against the behaviour documented in spaCy's own tests and docs
(tests/test_host_logic.py).  When fastai + spaCy are importable the reference's own tokenizer is used instead
(inference.py: ``learn.data.one_item``).
"""
from __future__ import annotations

import re
from typing import Dict, Iterable, List, Optional

# ---------------------------------------------------------------------------------------------- character classes
_ALPHA_LOWER = "a-zà-öø-ÿа-яёα-ωά-ώ"
_ALPHA_UPPER = "A-ZÀ-ÖØ-ÞА-ЯЁΑ-ΩΆ-Ώ"
_ALPHA = _ALPHA_LOWER + _ALPHA_UPPER
_HYPHENS = r"-|–|—|--|---|——|~"
_QUOTE_CHARS = "'\"”“`‘´’‚,„»«「」『』（）〔〕【】《》〈〉"
_CONCAT_QUOTES = "'\"”“`‘´’‚„»«"
_PUNCT = [r"…", r"……", r",", r":", r";", r"\!", r"\?", r"¿", r"؟", r"¡", r"\(", r"\)", r"\[", r"\]", r"\{", r"\}", r"<",
          r">", r"_", r"#", r"\*", r"&", r"。", r"？", r"！", r"，", r"、", r"；", r"：", r"～", r"·", r"।", r"،", r"؛", r"٪"]
_PUNCT_CLASS = r"…,:;\!\?¿؟¡\(\)\[\]\{\}<>_#\*&。？！，、；：～·।،؛٪"
_ELLIPSES = [r"\.\.+", r"…"]
_QUOTES = [re.escape(c) for c in _QUOTE_CHARS]
_CURRENCY = [r"\$", r"£", r"€", r"¥", r"฿", r"US\$", r"C\$", r"A\$", r"₽", r"﷼", r"₴"]
_UNITS = ("km|km²|km³|m|m²|m³|dm|dm²|dm³|cm|cm²|cm³|mm|mm²|mm³|ha|µm|nm|yd|in|ft|kg|g|mg|µg|t|lb|oz|m/s|km/h|kmh|mph|"
          "hPa|Pa|mbar|mb|MB|kb|KB|gb|GB|tb|TB|T|G|M|K|%")
_ICONS = [r"[\u2600-\u27BF\U0001F300-\U0001FAFF\u2190-\u21FF\u2B00-\u2BFF]"]

_PREFIXES = [r"§", r"%", r"=", r"—", r"–", r"\+(?![0-9])"] + _PUNCT + _ELLIPSES + _QUOTES + _CURRENCY + _ICONS
_SUFFIXES = (_PUNCT + _ELLIPSES + _QUOTES + _ICONS + [r"'s", r"'S", r"’s", r"’S", r"—", r"–"] + [
    r"(?<=[0-9])\+",
    r"(?<=°[FfCcKk])\.",
    r"(?<=[0-9])(?:" + "|".join(_CURRENCY) + r")",
    r"(?<=[0-9])(?:" + _UNITS + r")",
    r"(?<=[0-9" + _ALPHA_LOWER + r"%²\-\+" + _PUNCT_CLASS + re.escape(_CONCAT_QUOTES) + r"])\.",
    r"(?<=[" + _ALPHA_UPPER + r"][" + _ALPHA_UPPER + r"])\.",
])
_INFIXES = _ELLIPSES + _ICONS + [
    r"(?<=[0-9])[+\-\*^](?=[0-9-])",
    r"(?<=[" + _ALPHA_LOWER + re.escape(_CONCAT_QUOTES) + r"])\.(?=[" + _ALPHA_UPPER + re.escape(_CONCAT_QUOTES) + r"])",
    r"(?<=[" + _ALPHA + r"]),(?=[" + _ALPHA + r"])",
    r"(?<=[" + _ALPHA + r"])(?:" + _HYPHENS + r")(?=[" + _ALPHA + r"])",
    r"(?<=[" + _ALPHA + r"0-9])[:<>=/](?=[" + _ALPHA + r"])",
]
# longest alternative first, as spaCy's compile_prefix_regex / compile_suffix_regex do
_PREFIX_RE = re.compile("|".join("^" + p for p in sorted(_PREFIXES, key=len, reverse=True)))
_SUFFIX_RE = re.compile("|".join(p + "$" for p in sorted(_SUFFIXES, key=len, reverse=True)))
_INFIX_RE = re.compile("|".join(_INFIXES))
# token_match: URLs and things that look like them stay whole (spaCy's URL_PATTERN, abridged to scheme or www / domain.tld)
_URL_RE = re.compile(r"^(?:(?:https?|ftp)://\S+|www\.\S+|[\w.+-]+@[\w-]+(?:\.[\w-]+)+|(?:[\w-]+\.)+(?:com|org|net|io|dev|edu|gov)(?:/\S*)?)$",
                     re.IGNORECASE)


# ---------------------------------------------------------------------------------------------- special cases
def _english_exceptions() -> Dict[str, List[str]]:
    exc: Dict[str, List[str]] = {}

    def add(orth: str, pieces: List[str]):
        assert "".join(pieces) == orth, (orth, pieces)
        for variant, vp in ((orth, pieces), (orth[0].upper() + orth[1:], None)):
            if vp is None:  # capitalised variant: same split lengths
                vp, pos = [], 0
                for p in pieces:
                    vp.append(variant[pos:pos + len(p)])
                    pos += len(p)
            exc.setdefault(variant, vp)

    excluded = {"Ill", "ill", "Its", "its", "Hell", "hell", "Shell", "shell", "Shed", "shed", "were", "Were", "Well",
                "well", "Whore", "whore"}
    for pron in ("i",):
        for apo in ("'", "’", ""):
            add(pron + apo + "m", [pron, apo + "m"])
            add(pron + apo + "ma", [pron, apo + "m", "a"])
    for pron in ("i", "you", "he", "she", "it", "we", "they"):
        for apo in ("'", "’", ""):
            for tail in (["ll"], ["ll", "ve"], ["d"], ["d", "ve"]):
                pieces = [pron] + [apo + t for t in tail]
                orth = "".join(pieces)
                if orth not in excluded:
                    add(orth, pieces)
    for pron in ("i", "you", "we", "they"):
        for apo in ("'", "’", ""):
            add(pron + apo + "ve", [pron, apo + "ve"])
    for pron in ("you", "we", "they"):
        for apo in ("'", "’", ""):
            orth = pron + apo + "re"
            if orth not in excluded:
                add(orth, [pron, apo + "re"])
    for pron in ("he", "she", "it"):
        for apo in ("'", "’", ""):
            orth = pron + apo + "s"
            if orth not in excluded:
                add(orth, [pron, apo + "s"])
    for word in ("who", "what", "when", "where", "why", "how", "there", "that"):
        for apo in ("'", "’", ""):
            for tail in (["s"], ["ll"], ["ll", "ve"], ["re"], ["ve"], ["d"], ["d", "ve"]):
                if apo == "" and tail == ["s"] and word in ("who", "what", "when", "where", "why", "how", "there", "that"):
                    continue  # "whos", "whats" ... are not split
                pieces = [word] + [apo + t for t in tail]
                orth = "".join(pieces)
                if orth not in excluded:
                    add(orth, pieces)
    for verb in ("ca", "could", "do", "does", "did", "had", "may", "might", "must", "need", "ought", "sha", "should", "wo",
                 "would", "ai", "are", "is", "was", "were", "have", "has", "dare"):
        for nt in ("n't", "n’t", "nt"):
            orth = verb + nt
            if orth in excluded:
                continue
            add(orth, [verb, nt])
            if verb in ("could", "might", "must", "should", "would"):
                for apo in ("'", "’", ""):
                    add(orth + apo + "ve", [verb, nt, apo + "ve"])
    for verb in ("could", "might", "must", "should", "would"):
        for apo in ("'", "’", ""):
            add(verb + apo + "ve", [verb, apo + "ve"])
    for orth, pieces in (("let's", ["let", "'s"]), ("let’s", ["let", "’s"]), ("cannot", ["can", "not"]),
                         ("gonna", ["gon", "na"]), ("gotta", ["got", "ta"]), ("y'all", ["y'", "all"]),
                         ("y’all", ["y’", "all"]), ("'cause", ["'cause"]), ("ma'am", ["ma'am"]), ("o'clock", ["o'clock"]),
                         ("'em", ["'em"]), ("'til", ["'til"]), ("c'mon", ["c'm", "on"])):
        add(orth, pieces)
    for abbr in ("a.m.", "p.m.", "e.g.", "i.e.", "vs.", "v.s.", "Mr.", "Mrs.", "Ms.", "Dr.", "Prof.", "Jr.", "Sr.", "St.", "Mt.",
                 "Inc.", "Ltd.", "Co.", "Corp.", "Bros.", "Gen.", "Gov.", "Rep.", "Sen.", "Rev.", "Adm.", "Messrs.",
                 "Jan.", "Feb.", "Mar.", "Apr.", "Jun.", "Jul.", "Aug.", "Sep.", "Sept.", "Oct.", "Nov.", "Dec.",
                 "Ala.", "Ariz.", "Ark.", "Calif.", "Colo.", "Conn.", "Del.", "Fla.", "Ga.", "Ill.", "Ind.", "Kan.",
                 "Kans.", "Ky.", "La.", "Mass.", "Mich.", "Minn.", "Miss.", "Mo.", "Mont.", "Neb.", "Nebr.", "Nev.",
                 "Okla.", "Ore.", "Pa.", "Tenn.", "Va.", "Wash.", "Wis.", "N.Y.", "N.J.", "N.H.", "N.C.", "N.D.", "N.M.",
                 "S.C.", "S.D.", "D.C.", "U.S.", "U.K.", "U.N.", "E.U.", "p.s.", "P.S."):
        exc.setdefault(abbr, [abbr])
    for c in "abcdefghijklmnopqrstuvwxyz":
        exc.setdefault(c + ".", [c + "."])
        exc.setdefault(c.upper() + ".", [c.upper() + "."])
    for emo in (":)", ":-)", ":(", ":-(", ";)", ";-)", ":D", ":-D", ":P", ":-P", ":p", ":-p", ":o", ":O", ":/", ":-/", ":'(",
                ":|", ":-|", "<3", "</3", "^_^", "-_-", "o_o", "O_O", "o.O", "O.o", "xD", "XD", "(:", "):", "=)", "=(",
                ":3", ">:(", ":-*", ":*", ":>", ":]", ":[", "8)", "8-)", "\\o/", "¯\\_(ツ)_/¯"):
        exc.setdefault(emo, [emo])
    return exc


_EXCEPTIONS = _english_exceptions()


class SpacyLikeTokenizer:
    """``tokenizer(text) -> List[str]`` following spaCy 2.x ``Tokenizer.__call__`` / ``_tokenize`` / ``_split_affixes``
    / ``_attach_tokens``.  ``special_cases`` adds strings that must stay single tokens (fastai registers its
    ``text_spec_tok`` -- xxunk, xxpad, xxbos, xxfld, xxmaj, xxup, xxrep, xxwrep -- this way)."""

    def __init__(self, special_cases: Optional[Iterable[str]] = None):
        self.exceptions = dict(_EXCEPTIONS)
        for s in special_cases or ():
            self.exceptions[s] = [s]

    # spaCy tokenizer.pyx: Tokenizer.__call__
    def __call__(self, text: str) -> List[str]:
        out: List[str] = []
        if not text:
            return out
        i, start, in_ws = 0, 0, text[0].isspace()
        for i, ch in enumerate(text):
            if ch.isspace() != in_ws:
                if start < i:
                    span = text[start:i]
                    if in_ws:
                        out.append(span)           # a run of whitespace other than one separating space is a token
                    else:
                        out.extend(self._tokenize(span))
                if ch == " ":
                    start = i + 1                  # the single separating space belongs to the previous token
                else:
                    start = i
                in_ws = not in_ws
        if start < len(text):
            span = text[start:]
            if in_ws:
                out.append(span)
            else:
                out.extend(self._tokenize(span))
        return out

    # spaCy tokenizer.pyx: _tokenize -> _split_affixes + _attach_tokens
    def _tokenize(self, span: str) -> List[str]:
        prefixes: List[str] = []
        suffixes: List[str] = []
        s = span
        special: Optional[List[str]] = None
        last = None
        while s and s != last:
            last = s
            if s in self.exceptions:
                special = self.exceptions[s]
                break
            if _URL_RE.match(s):
                break
            m = _PREFIX_RE.search(s)
            if m and m.end() > 0:
                pre_len = m.end()
                minus_pre = s[pre_len:]
                if minus_pre and minus_pre in self.exceptions:   # special case after stripping the prefix
                    prefixes.append(s[:pre_len])
                    s = minus_pre
                    special = self.exceptions[s]
                    break
            else:
                pre_len = 0
            m2 = _SUFFIX_RE.search(s)
            if m2 and m2.start() < len(s):
                suf_len = len(s) - m2.start()
                minus_suf = s[:-suf_len]
                if minus_suf and minus_suf in self.exceptions:
                    suffixes.append(s[-suf_len:])
                    s = minus_suf
                    special = self.exceptions[s]
                    break
            else:
                suf_len = 0
            if pre_len and suf_len and pre_len + suf_len <= len(s):
                prefixes.append(s[:pre_len])
                suffixes.append(s[-suf_len:])
                s = s[pre_len:len(s) - suf_len]
            elif pre_len:
                prefixes.append(s[:pre_len])
                s = s[pre_len:]
            elif suf_len:
                suffixes.append(s[-suf_len:])
                s = s[:-suf_len]
        toks = list(prefixes)
        if s:
            if special is not None:
                toks.extend(special)
            elif s in self.exceptions:
                toks.extend(self.exceptions[s])
            elif _URL_RE.match(s):
                toks.append(s)
            else:
                pos = 0
                for m in _INFIX_RE.finditer(s):
                    if m.start() == m.end():
                        continue
                    if m.start() > pos:
                        toks.append(s[pos:m.start()])
                    toks.append(m.group())
                    pos = m.end()
                if pos < len(s):
                    toks.append(s[pos:])
        toks.extend(reversed(suffixes))
        return [t for t in toks if t]
