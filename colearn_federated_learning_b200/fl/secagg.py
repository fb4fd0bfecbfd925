"""Secure aggregation of the device updates in remote mode (Bonawitz et al., "Practical Secure Aggregation for
Privacy-Preserving Machine Learning", CCS 2017): the coordinator learns the sum of the devices' deltas and nothing about any
one of them, and devices that drop out before they send their masked update are tolerated.

Threat model: an honest-but-curious coordinator (it follows the protocol but tries to learn individual updates from what it
receives) and anyone who reads the wire.  Not covered: a coordinator that lies (for example by sending different survivor
sets to different devices: Bonawitz's consistency round and signatures are not built), collusion between the coordinator and
devices, timing side channels of the Python key agreement, the loss and sample count a reply carries in the clear, and a
device that sends a wrong mask or seed (it corrupts the aggregate; the ring bounds the damage, see :func:`frac_bits`).

Protocol (``U1_t``: the devices asked to fit in round ``t``; ``U2_t``: those whose masked reply passed the checks; ``D_t =
U1_t \\ U2_t``):

1. Setup, once per training: every device makes a fresh Diffie-Hellman key pair in the RFC 7919 ``ffdhe2048`` group (256-bit
   private exponent) for the training's tag and returns its public key; a second setup message gives every device the key
   list in setup order.  Each pair derives ``s_uv = HKDF-SHA256(DH(u, v), info = tag | both ids in setup order)``.
2. Round ``t``: the fit request carries the tag, ``t``, ``U1_t``, the clip ``C`` and the fraction bits ``f``.  The device
   derives the round's pair seeds ``s_uv^t = HKDF(s_uv, "round t")``, draws a fresh self seed ``b_u^t``, fits, and replies
   ``y_u = enc(d_u) + PRG(b_u^t) + sum_{v in U1_t} +-PRG(s_uv^t)`` (mod 2^32; ``+`` when ``u`` comes before ``v`` in the
   setup order): ``4 P`` bytes, plus the counts of clipped and non-finite coordinates.
3. Unmask: each device of ``U2_t`` reveals ``b_u^t`` and ``s_uv^t`` for ``v in D_t``, once per round and only for
   ``|U2_t| >= 2``; the coordinator removes those streams from ``sum_{U2} y_u`` and applies the decoded mean.  If a device of
   ``U2_t`` does not answer, the round is abandoned (theta unchanged): asking again after a partial unmask would expose the
   devices that did answer.

The arithmetic (ChaCha20 streams, the fixed-point code) is ``ops/csrc/secagg.cuh``; ``ops.reference`` transcribes it.
"""
from __future__ import annotations

import hashlib
import hmac
import math
import secrets
from dataclasses import dataclass, field
from fractions import Fraction
from typing import Any, Dict, List, Sequence, Tuple

import numpy as np

# RFC 7919 ffdhe2048: p = 2^2048 - 2^1984 + (floor(2^1918 e) + 560316) 2^64 - 1, generator 2 of the subgroup of order q = (p - 1) / 2
P = int(
    "FFFFFFFFFFFFFFFFADF85458A2BB4A9AAFDC5620273D3CF1D8B9C583CE2D3695"
    "A9E13641146433FBCC939DCE249B3EF97D2FE363630C75D8F681B202AEC4617A"
    "D3DF1ED5D5FD65612433F51F5F066ED0856365553DED1AF3B557135E7F57C935"
    "984F0C70E0E68B77E2A689DAF3EFE8721DF158A136ADE73530ACCA4F483A797A"
    "BC0AB182B324FB61D108A94BB2C8E3FBB96ADAB760D7F4681D4F42A3DE394DF4"
    "AE56EDE76372BB190B07A7C8EE0A6D709E02FCE1CDF7E2ECC03404CD28342F61"
    "9172FE9CE98583FF8E4F1232EEF28183C3FE3B1B4C6FAD733BB5FCBC2EC22005"
    "C58EF1837D1683B2C6F34A26C1B2EFFA886B423861285C97FFFFFFFFFFFFFFFF", 16)
Q = (P - 1) // 2
G = 2
PK_BYTES = 256
SEED_BYTES = 32
SUM_MAX = (1 << 31) - 1          # the largest honest |sum| of codes: an int32 never wraps
MAX_FRAC_BITS = 64


# ---- primitives --------------------------------------------------------------------------------------------------------------
def hkdf_sha256(ikm: bytes, info: bytes, length: int = SEED_BYTES, salt: bytes = b"") -> bytes:
    """RFC 5869 HKDF with SHA-256 (an empty salt is HashLen zero bytes)."""
    prk = hmac.new(salt or bytes(32), ikm, hashlib.sha256).digest()
    out, block = b"", b""
    for i in range(1, -(-length // 32) + 1):
        block = hmac.new(prk, block + info + bytes([i]), hashlib.sha256).digest()
        out += block
    return out[:length]


def check_public_key(pk: int) -> int:
    """``pk`` if it is an element of the order-q subgroup other than 1 (``2 <= pk <= p - 2`` and ``pk^q = 1 mod p``), else
    ValueError: a peer's key is untrusted input."""
    if not isinstance(pk, int) or not 2 <= pk <= P - 2 or pow(pk, Q, P) != 1:
        raise ValueError("public key outside the ffdhe2048 prime-order subgroup")
    return pk


def pk_to_bytes(pk: int) -> bytes:
    return pk.to_bytes(PK_BYTES, "big")


def pk_from_bytes(b: Any) -> int:
    if not isinstance(b, bytes) or len(b) != PK_BYTES:
        raise ValueError(f"public key of {len(b) if isinstance(b, bytes) else None} bytes, expected {PK_BYTES}")
    return check_public_key(int.from_bytes(b, "big"))


@dataclass(frozen=True)
class KeyPair:
    sk: int
    pk: int

    @staticmethod
    def generate() -> "KeyPair":
        sk = 0
        while sk < 2:
            sk = secrets.randbits(256)
        return KeyPair(sk, pow(G, sk, P))


def pair_seed(sk: int, peer_pk: int, tag: str, first: str, second: str) -> bytes:
    """``s_uv``: HKDF of the Diffie-Hellman secret with the peer, bound to the training's tag and the two ids in setup order"""
    z = pow(check_public_key(peer_pk), sk, P)
    return hkdf_sha256(z.to_bytes(PK_BYTES, "big"), f"colearn secagg|{tag}|{first}|{second}".encode())


def round_seed(seed: bytes, t: int) -> bytes:
    """``s_uv^t``: revealing one round's seed unmasks no other round"""
    return hkdf_sha256(seed, f"round {int(t)}".encode())


def code_bound(clip: float, f: int) -> int:
    """``ceil(C 2^f)`` with ``C`` rounded to float32 as the kernel clamps: the largest |code| of one device"""
    return math.ceil(Fraction(float(np.float32(clip))) * (1 << f))


def frac_bits(clip: float, devices: int) -> int:
    """The largest ``f`` (at most 64) with ``devices * ceil(C 2^f) <= 2^31 - 1``: no honest sum of that many codes wraps.
    Whatever any device sends, the decoded mean of ``n`` survivors stays within ``2^31 2^-f / n``, about ``C devices / n``."""
    check_clip(clip)
    if devices < 1 or devices * code_bound(clip, 0) > SUM_MAX:
        raise ValueError(f"a clip of {clip} leaves no fraction bits for {devices} devices")
    f = 0
    while f < MAX_FRAC_BITS and devices * code_bound(clip, f + 1) <= SUM_MAX:
        f += 1
    return f


def check_clip(clip: Any) -> float:
    """``clip`` as a float if it is finite and > 0 in float32 too (the kernel clamps in float32), else ValueError"""
    ok = not isinstance(clip, bool) and isinstance(clip, (int, float)) and math.isfinite(clip) and clip > 0
    if ok:
        with np.errstate(over="ignore"):
            ok = bool(np.float32(clip) > 0 and np.isfinite(np.float32(clip)))
    if not ok:
        raise ValueError(f"the secure-aggregation clip must be finite and > 0, not {clip!r}")
    return float(clip)


def pair_sign(order: Sequence[str], u: str, v: str) -> int:
    """+1 when ``u`` comes before ``v`` in the setup order, -1 otherwise: the pair masks cancel in the sum"""
    return 1 if order.index(u) < order.index(v) else -1


# ---- checks of untrusted replies on the coordinator ----------------------------------------------------------------------------
def check_masked_reply(update: Dict[str, Any], p: int) -> Tuple[np.ndarray, int, int]:
    """``(masked uint32 [p], clipped, nonfinite)`` of a device's masked reply, or ValueError: exactly ``4 p`` bytes and counts
    that are ints in ``[0, p]``."""
    if update.get("secagg") != "masked":
        raise ValueError(f"reply {update.get('secagg')!r} returned, a masked update asked for")
    masked = update.get("masked")
    if not isinstance(masked, bytes) or len(masked) != 4 * p:
        raise ValueError(f"masked update of {len(masked) if isinstance(masked, bytes) else None} bytes, expected {4 * p}")
    counts = [update.get("clipped"), update.get("nonfinite")]
    if any(type(c) is not int or not 0 <= c <= p for c in counts):
        raise ValueError(f"clipped / non-finite counts {counts} outside 0..{p}")
    return np.frombuffer(masked, dtype="<u4").astype(np.uint32), counts[0], counts[1]


def check_unmask_reply(resp: Dict[str, Any], dropped: Sequence[str]) -> Tuple[bytes, Dict[str, bytes]]:
    """``(self seed, {dropped peer: pair seed})`` of an unmask reply, or ValueError: 32-byte seeds, exactly one per asked pair."""
    own, pairs = resp.get("self_seed"), resp.get("pair_seeds")
    if not isinstance(own, bytes) or len(own) != SEED_BYTES:
        raise ValueError("self seed missing or not 32 bytes")
    if not isinstance(pairs, dict) or sorted(pairs) != sorted(dropped):
        raise ValueError(f"pair seeds for {sorted(pairs) if isinstance(pairs, dict) else None}, asked for {sorted(dropped)}")
    if any(not isinstance(s, bytes) or len(s) != SEED_BYTES for s in pairs.values()):
        raise ValueError("pair seed not 32 bytes")
    return own, dict(pairs)


def correction_streams(order: Sequence[str], survivors: Sequence[str], dropped: Sequence[str],
                       seeds: Dict[str, Tuple[bytes, Dict[str, bytes]]]) -> Tuple[List[bytes], List[int]]:
    """The streams the coordinator adds to ``sum_{U2} y_u``: ``-PRG(b_u)`` for every survivor and ``-+PRG(s_uv)`` for every
    survivor ``u`` and dropped ``v`` (the opposite of the sign ``u`` masked with)."""
    keys, signs = [], []
    for u in survivors:
        own, pairs = seeds[u]
        keys.append(own)
        signs.append(-1)
        for v in dropped:
            keys.append(pairs[v])
            signs.append(-pair_sign(order, u, v))
    return keys, signs


# ---- device side ---------------------------------------------------------------------------------------------------------------
@dataclass
class _Training:
    keys: KeyPair
    me: str = ""
    order: List[str] = field(default_factory=list)
    seeds: Dict[str, bytes] = field(default_factory=dict)       # peer -> s_uv
    revealed: set = field(default_factory=set)                   # peers whose seeds this device gave away
    last_round: int = -1
    rounds: Dict[int, Dict[str, Any]] = field(default_factory=dict)   # t -> {"u1", "self", "answered"}


class SecAggDevice:
    """A device's secure-aggregation state, per training tag, in memory only: the key pair, the pair seeds, the peers whose
    seeds it revealed (refused in any later round) and, per round, its self seed and whether it answered the unmask."""
    KEEP = 4                      # trainings remembered (a new setup forgets the oldest)

    def __init__(self) -> None:
        self._t: Dict[str, _Training] = {}

    def setup(self, tag: str) -> bytes:
        if not isinstance(tag, str) or not tag:
            raise ValueError("secure aggregation setup without a tag")
        while len(self._t) >= self.KEEP:
            self._t.pop(next(iter(self._t)))
        self._t[tag] = _Training(KeyPair.generate())
        return pk_to_bytes(self._t[tag].keys.pk)

    def learn_peers(self, tag: str, ids: Sequence[str], pks: Sequence[bytes]) -> str:
        """Takes the key list of the training (setup order), finds this device by its own public key and derives the pair
        seeds; returns this device's id"""
        tr = self._training(tag)
        if tr.order:
            raise ValueError("the peers of this training are already known")
        if not isinstance(ids, list) or not isinstance(pks, list) or len(ids) != len(pks) or len(set(ids)) != len(ids) or \
                any(not isinstance(i, str) for i in ids):
            raise ValueError("malformed peer list")
        mine = pk_to_bytes(tr.keys.pk)
        if pks.count(mine) != 1:
            raise ValueError("this device's public key is not in the peer list")
        me = ids[pks.index(mine)]
        seeds = {}
        for i, (v, pk) in enumerate(zip(ids, pks)):
            if v != me:
                first, second = (me, v) if ids.index(me) < i else (v, me)
                seeds[v] = pair_seed(tr.keys.sk, pk_from_bytes(pk), tag, first, second)
        tr.me, tr.order, tr.seeds = me, list(ids), seeds
        return me

    def begin_round(self, tag: str, t: int, u1: Sequence[str], clip: float, f: int) -> Tuple[List[bytes], List[int]]:
        """Checks round ``t``'s request and returns this device's mask streams (its fresh self seed first, then one pair
        seed per other participant) and their signs"""
        tr = self._training(tag)
        if not tr.order:
            raise ValueError("fit before the peers of this training are known")
        if type(t) is not int or t <= tr.last_round:
            raise ValueError(f"round {t!r} is not after round {tr.last_round}")
        if not isinstance(u1, list) or len(set(u1)) != len(u1) or len(u1) < 2 or tr.me not in u1:
            raise ValueError("the participant list must name this device and at least one other, once each")
        unknown = [v for v in u1 if v not in tr.order]
        if unknown:
            raise ValueError(f"unknown participants {unknown}")
        again = [v for v in u1 if v in tr.revealed]
        if again:
            raise ValueError(f"participants {again} were reported dropped earlier: their pair seeds are revealed")
        check_clip(clip)
        if type(f) is not int or not 0 <= f <= MAX_FRAC_BITS or len(u1) * code_bound(clip, f) > SUM_MAX:
            raise ValueError(f"{f!r} fraction bits let a sum of {len(u1)} codes wrap")
        own = secrets.token_bytes(SEED_BYTES)
        keys, signs = [own], [1]
        for v in u1:
            if v != tr.me:
                keys.append(round_seed(tr.seeds[v], t))
                signs.append(pair_sign(tr.order, tr.me, v))
        tr.last_round = t
        tr.rounds = {t: {"u1": list(u1), "self": own, "answered": False}}   # an earlier round can no longer be unmasked
        return keys, signs

    def unmask(self, tag: str, t: int, u2: Sequence[str]) -> Dict[str, Any]:
        """The seeds of round ``t`` for the survivors ``u2``: the self seed and the pair seeds of the dropped participants,
        once per round, only if this device survived and at least two did"""
        tr = self._training(tag)
        rnd = tr.rounds.get(t) if type(t) is int else None
        if rnd is None:
            raise ValueError(f"no round {t!r} to unmask")
        if rnd["answered"]:
            raise ValueError(f"round {t} was unmasked already")
        if not isinstance(u2, list) or len(set(u2)) != len(u2) or len(u2) < 2 or tr.me not in u2 or \
                any(v not in rnd["u1"] for v in u2):
            raise ValueError("the survivors must be at least two participants of the round, this device among them")
        rnd["answered"] = True
        dropped = [v for v in rnd["u1"] if v not in u2]
        tr.revealed.update(dropped)
        return {"self_seed": rnd["self"], "pair_seeds": {v: round_seed(tr.seeds[v], t) for v in dropped}}

    def _training(self, tag: Any) -> _Training:
        tr = self._t.get(tag) if isinstance(tag, str) else None
        if tr is None:
            raise ValueError(f"no secure-aggregation setup for tag {tag!r}")
        return tr
