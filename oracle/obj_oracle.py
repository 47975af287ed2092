"""TEST INFRASTRUCTURE ONLY -- Python twins of the device OBJ reader's rules (disn_b200/csrc/obj_read.cu): the line and
token split, the coordinate grammar and the rule that decides which coordinates the device computes itself.  The
specification the reader must match is create_sdf.read_obj / read_obj_parts; tests compare these twins with it."""
import re

SEPARATORS = b" \t\v\f\x1c\x1d\x1e\x1f"      # str.split()'s ASCII whitespace within a line
COORD = re.compile(rb"[+-]?(?:[0-9]+(?:\.[0-9]*)?|\.[0-9]+)(?:[eE][+-]?[0-9]+)?\Z")
SPECIAL = re.compile(rb"[+-]?(?:inf|infinity|nan)\Z", re.IGNORECASE)
_SPLIT = re.compile(b"[" + re.escape(SEPARATORS) + b"]+")


def lines(data: bytes):
    """The lines of a file as the device finds them: a line ends at "\\n", "\\r\\n" or a lone "\\r"; a last line
    without an end is a line.  Each line is returned without its end."""
    out, start, i, n = [], 0, 0, len(data)
    while i < n:
        ch = data[i:i + 1]
        if ch == b"\n" or ch == b"\r":
            out.append(data[start:i])
            i += 2 if data[i:i + 2] == b"\r\n" else 1
            start = i
        else:
            i += 1
    if start < n:
        out.append(data[start:])
    return out


def tokens(line: bytes):
    return [t for t in _SPLIT.split(line) if t]


def is_coordinate(tok: bytes) -> bool:
    return bool(COORD.match(tok) or SPECIAL.match(tok))


def fast_value(tok: bytes):
    """The float64 the device computes for a coordinate token, or None when it leaves the token to the host: a
    significand of at most 19 significant digits and at most 2^53, and a decimal exponent within +-22, give one
    correctly rounded multiply or divide by an exact power of ten."""
    if not COORD.match(tok):
        return None
    neg = tok[:1] == b"-"
    body = tok.lstrip(b"+-")
    mant, _, exp = body.lower().partition(b"e")
    ip, _, fp = mant.partition(b".")
    digits = (ip + fp).lstrip(b"0")
    if len(digits) > 19:
        return None
    m, e = int(digits or b"0"), int(exp or b"0") - len(fp)
    if m > 2 ** 53 or abs(e) > 22:
        return None
    v = float(m) * 10.0 ** e if e >= 0 else float(m) / 10.0 ** -e
    return -v if neg else v
