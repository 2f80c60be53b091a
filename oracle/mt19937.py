"""MT19937 exactly as CPython's ``random`` module drives it.  TEST INFRASTRUCTURE (see oracle/__init__.py).

The reference's ``Squared.reset`` draws its target with ``random.sample(possible_targets, 1)`` from the
process-global ``random`` after ``random.seed(seed)`` (reference pufferlib/environments/ocean/ocean.py:448-461).
For an int seed CPython's ``random.seed`` is ``init_by_array(key)`` with ``key`` = the little-endian 32-bit
words of ``abs(seed)`` (one word for seed < 2**32), and ``random.sample(pop, 1)`` with ``len(pop) == 24`` is one
``_randbelow_with_getrandbits(24)``: ``r = getrandbits(5)`` (= ``genrand_uint32() >> 27``) repeated until
``r < 24``.  ``tests/test_oracle_mt19937.py`` checks this file against ``random`` itself.
"""

N, M = 624, 397
MATRIX_A, UPPER, LOWER = 0x9908B0DF, 0x80000000, 0x7FFFFFFF
MASK32 = 0xFFFFFFFF


class MT19937:
    def __init__(self, seed=None):
        self.mt = [0] * N
        self.idx = N + 1
        if seed is not None:
            self.seed(seed)

    def init_genrand(self, s):
        mt = self.mt
        mt[0] = s & MASK32
        for i in range(1, N):
            mt[i] = (1812433253 * (mt[i - 1] ^ (mt[i - 1] >> 30)) + i) & MASK32
        self.idx = N

    def init_by_array(self, key):
        self.init_genrand(19650218)
        mt = self.mt
        i, j = 1, 0
        klen = len(key)
        for _ in range(max(N, klen)):
            mt[i] = ((mt[i] ^ ((mt[i - 1] ^ (mt[i - 1] >> 30)) * 1664525)) + key[j] + j) & MASK32
            i += 1
            j += 1
            if i >= N:
                mt[0] = mt[N - 1]
                i = 1
            if j >= klen:
                j = 0
        for _ in range(N - 1):
            mt[i] = ((mt[i] ^ ((mt[i - 1] ^ (mt[i - 1] >> 30)) * 1566083941)) - i) & MASK32
            i += 1
            if i >= N:
                mt[0] = mt[N - 1]
                i = 1
        mt[0] = 0x80000000
        self.idx = N

    def seed(self, s):
        """``random.seed(int)``: key = 32-bit little-endian words of abs(s) (at least one word)."""
        s = abs(int(s))
        key = []
        while s:
            key.append(s & MASK32)
            s >>= 32
        self.init_by_array(key or [0])

    def _twist(self):
        mt = self.mt
        for k in range(N):
            y = (mt[k] & UPPER) | (mt[(k + 1) % N] & LOWER)
            mt[k] = mt[(k + M) % N] ^ (y >> 1) ^ (MATRIX_A if y & 1 else 0)
        self.idx = 0

    def genrand_uint32(self):
        if self.idx >= N:
            self._twist()
        y = self.mt[self.idx]
        self.idx += 1
        y ^= y >> 11
        y ^= (y << 7) & 0x9D2C5680
        y ^= (y << 15) & 0xEFC60000
        y ^= y >> 18
        return y & MASK32

    def getrandbits(self, k):
        assert 0 < k <= 32
        return self.genrand_uint32() >> (32 - k)

    def randbelow(self, n):
        k = int(n).bit_length()
        r = self.getrandbits(k)
        while r >= n:
            r = self.getrandbits(k)
        return r

    def copy(self):
        c = MT19937()
        c.mt = list(self.mt)
        c.idx = self.idx
        return c
