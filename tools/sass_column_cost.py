"""Static instruction cost of dp_pair's column bodies in k_populate_fast<B, 1>, read from the SASS: the steady body, the prologue
(the first 2B columns, entered at the column's first cell) and the epilogue (the last 2B-1 columns, left after the row-L cell),
per column and per cell pair, and the instructions one dp_pair call executes for a read length L. CPU only: it reads a cubin,
a shared library (both through cuobjdump) or a saved `cuobjdump -sass` listing.

usage: python tools/sass_column_cost.py <cubin | .so | listing> [--band 16] [--L 150] [--form oge|general] [--columns]

How it counts: the function's basic blocks are cut at branch targets and after branches. A cell is recognised by its row-entry
load (one LDS.64 per cell), the steady body as the block with 2B of them, the deletion-update form by its VIMNMX count (OGE: one
per cell, general: two). Every column x of a call is then walked through the control flow from the loop header to the loop's
back edge, counting instructions: compares of the column index with a constant are evaluated, an indexed branch (BRX) goes to
the prologue entry whose chain suffix has the cells column x runs, the epilogue's exit tests leave after the row-L cell, and a
branch that depends on L alone (x <= L) goes the way that reaches the column's body. Counts are static (every instruction
counted once per execution, predicated ones included); they are not a measurement of time.
"""
import argparse
import re
import subprocess
import sys

BRANCH = re.compile(r"\b(BRA|BRX|EXIT|RET|JMP|JMX)\b")


def cuobjdump():
    """cuobjdump next to the nvcc the build uses (NVCC, /usr/local/cuda/bin), else the one on PATH"""
    import os
    for nvcc in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc"):
        if nvcc and os.path.isabs(nvcc):
            cand = os.path.join(os.path.dirname(nvcc), "cuobjdump")
            if os.path.exists(cand):
                return cand
    return "cuobjdump"


def listing(path):
    with open(path, "rb") as f:
        head = f.read(4)
    if head == b"\x7fELF":
        return subprocess.run([cuobjdump(), "-sass", path], capture_output=True, text=True, check=True).stdout
    with open(path) as f:
        return f.read()


def function(text, band):
    for part in text.split("Function : ")[1:]:
        name = part.split("\n")[0].strip()
        if "k_populate_fastILi%dELi1E" % band in name:
            ins = []
            for line in part.split("\n"):
                m = re.match(r"^\s+/\*([0-9a-f]+)\*/\s+(.*?)\s*;", line)
                if m:
                    ins.append((int(m.group(1), 16), m.group(2).strip().replace(".reuse", "")))
            return name, ins
    sys.exit("no k_populate_fast<%d, 1> in the input" % band)


class Block:
    def __init__(self, ins):
        self.ins = ins
        self.addr = ins[0][0]
        self.n = len(ins)
        self.lds = sum("LDS.64" in t for _, t in ins)
        self.vimnmx = sum(re.match(r"(@!?P\d+ )?VIMNMX\.", t) is not None for _, t in ins)
        self.movs = sum(re.match(r"(@!?P\d+ )?(IMAD\.)?MOV", t) is not None for _, t in ins)
        last = ins[-1][1]
        self.last = last
        m = re.search(r"\b(BRA|BRX)\b.*?(0x[0-9a-f]+)\s*$", last)
        self.target = int(m.group(2), 16) if m and "BRX" not in last else None
        self.cond = re.match(r"@!?P\d+ ", last) is not None
        self.brx = "BRX" in last
        self.ends = BRANCH.search(last) is not None


def blocks_of(ins):
    targets = set()
    for _, t in ins:
        m = re.search(r"\bBRA\b.*?(0x[0-9a-f]+)\s*$", t)
        if m:
            targets.add(int(m.group(1), 16))
    out, cur = [], []
    for a, t in ins:
        if a in targets and cur:
            out.append(Block(cur)); cur = []
        cur.append((a, t))
        if BRANCH.search(t):
            out.append(Block(cur)); cur = []
    if cur:
        out.append(Block(cur))
    return out


class Cfg:
    def __init__(self, blocks, K, form):
        self.b = blocks
        self.K = K
        self.at = {b.addr: i for i, b in enumerate(blocks)}
        steady = sorted((b.vimnmx, i) for i, b in enumerate(blocks) if b.lds == K)
        if len(steady) < 2:
            sys.exit("expected two steady bodies (OGE and general form) with %d LDS.64 each, found %d" % (K, len(steady)))
        self.steady = steady[0][1] if form == "oge" else steady[-1][1]
        per_cell = round(blocks[self.steady].vimnmx / K)
        self.cell = lambda i: blocks[i].lds == 1 and blocks[i].vimnmx == per_cell
        # epilogue: the longest run of cell blocks that each end in a conditional branch (the exit test), plus a last cell
        runs, r = [], []
        for i, b in enumerate(blocks):
            if self.cell(i) and b.cond and b.target is not None:
                r.append(i)
            else:
                if r and self.cell(i):
                    r.append(i)
                runs.append(r); r = []
        runs.append(r)
        self.exit_chain = max(runs, key=len)
        # the top cell (k = 2B-1) has no deletion update, so in the general form it has one VIMNMX less than the others
        first = self.exit_chain[0] if self.exit_chain else 0
        if len(self.exit_chain) == K - 2 and first > 0 and blocks[first - 1].lds == 1 and blocks[first - 1].cond:
            self.exit_chain.insert(0, first - 1)
        if len(self.exit_chain) not in (K - 1, K):      # cells 2B-1 .. 1, or .. 0 where the row-L test is also made for k = 0
            sys.exit("epilogue: found %d exit-test cells, expected %d" % (len(self.exit_chain), K - 1))
        # the DP loop: the narrowest backward branch whose range holds the steady body and the epilogue
        lo = min(blocks[self.steady].addr, blocks[self.exit_chain[0]].addr)
        hi = max(blocks[self.steady].addr, blocks[self.exit_chain[-1]].addr)
        loops = [(b.addr - b.target, i) for i, b in enumerate(blocks)
                 if b.target is not None and b.target <= lo and b.addr >= hi]
        if not loops:
            sys.exit("no loop around the steady body and the epilogue")
        self.latch = min(loops)[1]
        self.header = self.at[blocks[self.latch].target]
        # x: the register the header compares with 2B-1 or 2B
        self.xreg = None
        for i in range(self.header, self.steady):
            for _, t in blocks[i].ins:
                m = re.match(r"ISETP\.\w+(\.U32)?\.AND P\d+, PT, (R\d+), (0x[0-9a-f]+|\d+), PT", t)
                if m and int(m.group(3), 0) in (K - 1, K):
                    self.xreg = m.group(2)
                    break
            if self.xreg:
                break
        if self.xreg is None:
            sys.exit("no compare of the column index with 2B in the loop header")
        self.brx_entries = self._brx_entries()

    def succ(self, i):
        b = self.b[i]
        out = []
        if b.brx:
            out += [j for j, _ in self.brx_entries.get(i, [])]
        if b.target is not None and b.target in self.at:
            out.append(self.at[b.target])
        if (not b.ends or b.cond) and i + 1 < len(self.b):
            out.append(i + 1)
        return out

    def _brx_entries(self):
        """BRX successors: the blocks right after it up to the next BRX, each a prologue entry cell that branches into the chain.
        Every entry is keyed by the number of chain cells it runs after itself (x - 2 for column x)."""
        out = {}
        for i, b in enumerate(self.b):
            if not b.brx:
                continue
            ents, j = [], i + 1
            while j < len(self.b) and not self.b[j].brx and self.cell(j) and not self.b[j].cond and self.b[j].target is not None:
                ents.append((j, self._chain_len(self.at[self.b[j].target])))
                j += 1
            out[i] = ents
        return out

    def _chain_len(self, i):
        n = 0
        while i < len(self.b) and self.cell(i) and not self.b[i].cond and i not in self.exit_chain:
            n += 1
            if self.b[i].target is not None and self.b[i].ends:
                break
            i += 1
        return n

    def dist(self, src, dst):
        """Fewest instructions on a path src -> dst that does not pass the loop's back edge (None: no such path)."""
        import heapq
        best, heap = {src: 0}, [(0, src)]
        while heap:
            d, i = heapq.heappop(heap)
            if i == dst:
                return d
            if d > best.get(i, 1 << 60) or i == self.latch:
                continue
            for j in self.succ(i):
                nd = d + self.b[i].n
                if nd < best.get(j, 1 << 60):
                    best[j] = nd
                    heapq.heappush(heap, (nd, j))
        return None

    def walk(self, x, L):
        """Instructions executed by column x of a call with read length L: header to back edge."""
        K, b = self.K, self.b
        if x >= K and x <= L:
            goal = self.steady
        elif x > L:
            goal = self.exit_chain[0]
        else:
            goal = self.prologue_target(x)
        pred, i, count, steps = {}, self.header, 0, 0
        klo = x - L
        while True:
            steps += 1
            if steps > 10000:
                raise RuntimeError("walk did not end (x=%d)" % x)
            blk = b[i]
            count += blk.n
            for _, t in blk.ins:
                m = re.match(r"ISETP\.(\w+?)(\.U32)?\.AND (P\d+), PT, (R\d+), (0x[0-9a-f]+|-?\d+), PT", t)
                if m and m.group(4) == self.xreg:
                    c, v = m.group(1), int(m.group(5), 0)
                    pred[m.group(3)] = {"GT": x > v, "GE": x >= v, "LT": x < v, "LE": x <= v, "EQ": x == v, "NE": x != v}[c]
                else:               # any other write of a predicate: unknown from here on
                    d = re.match(r"^(?:@!?P\d+ )?[A-Z][\w.]* (P\d+), ", t)
                    if d:
                        pred.pop(d.group(1), None)
            if i == self.latch:
                return count
            if blk.brx:                     # the prologue dispatch: on to column x's entry cell
                i = goal
                continue
            if blk.target is not None and not blk.cond:
                i = self.at[blk.target]
                continue
            if blk.cond and blk.target is not None:
                if i in self.exit_chain:
                    take = self.exit_chain.index(i) == K - 1 - klo
                else:
                    m = re.match(r"@(!?)(P\d+) ", blk.last)
                    p = pred.get(m.group(2))
                    if p is not None:
                        take = p != (m.group(1) == "!")
                    else:           # depends on L: the nearer way to the column's body
                        dt = self.dist(self.at[blk.target], goal)
                        df = self.dist(i + 1, goal)
                        take = dt is not None and (df is None or dt < df)
                i = self.at[blk.target] if take else i + 1
                continue
            i += 1

    def prologue_target(self, x):
        """The first block of column x's cells: its entry cell after an indexed branch, or, where the dispatch jumps straight
        into the chain of fall-through cells (cells 2B-1 .. 0 in address order), chain cell x-1; for column 0 the chain's end."""
        if not hasattr(self, "_chain"):
            runs, r = [], []
            for i, b in enumerate(self.b):
                if self.cell(i) and not b.ends and i not in self.exit_chain:
                    r.append(i)
                else:
                    runs.append(r); r = []
            runs.append(r)
            self._chain = max(runs, key=len)
        # column x runs its entry cell x-1 and then x-1 chain cells; column 0 runs none and goes where column 1's entry goes
        ents = [j for e in self.brx_entries.values() for j, n in e if n == max(x - 1, 0)]
        if ents:
            return ents[0] if x > 0 else self.at[self.b[ents[0]].target]
        return self._chain[len(self._chain) - x] if x > 0 else self._chain[-1] + 1


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("input")
    ap.add_argument("--band", type=int, default=16)
    ap.add_argument("--L", type=int, default=150)
    ap.add_argument("--form", choices=["oge", "general"], default="oge")
    ap.add_argument("--columns", action="store_true", help="print the cost of every column")
    a = ap.parse_args()
    K = 2 * a.band
    if a.L < K - 1:
        sys.exit("--L must be at least 2B-1 (the short-read body is not modelled)")
    name, ins = function(listing(a.input), a.band)
    g = Cfg(blocks_of(ins), K, a.form)
    W = a.L + K - 1
    cost = [g.walk(x, a.L) for x in range(W + 1)]
    pro, steady, epi = cost[:K], cost[K:a.L + 1], cost[a.L + 1:]
    tri = K * (K - 1) // 2
    sb = g.b[g.steady]
    print("%s, %s form, band %d (2B = %d), L = %d" % (name, a.form, a.band, K, a.L))
    print("steady body   : %d instructions per %d cell pairs = %.2f per cell pair (%d moves); column with top and end: %d"
          % (sb.n, K, sb.n / K, sb.movs, steady[0] if steady else g.walk(K, K)))
    ec = [g.b[i].n for i in g.exit_chain]
    print("epilogue cells: %s  (max %d, moves %d)" % (" ".join(map(str, ec)), max(ec), sum(g.b[i].movs for i in g.exit_chain)))
    print("prologue      : %d columns, %d instructions for %d cell pairs = %.2f per cell pair" % (len(pro), sum(pro), tri, sum(pro) / tri))
    print("epilogue      : %d columns, %d instructions for %d cell pairs = %.2f per cell pair" % (len(epi), sum(epi), tri, sum(epi) / tri))
    print("steady        : %d columns, %d instructions for %d cell pairs = %.2f per cell pair"
          % (len(steady), sum(steady), K * len(steady), sum(steady) / max(1, K * len(steady))))
    print("per call      : %d instructions (prologue %d + steady %d + epilogue %d); at steady cost the ramps would be %d"
          % (sum(cost), sum(pro), sum(steady), sum(epi), round(2 * tri * (steady[0] if steady else 0) / K)))
    if a.columns:
        print("columns       : " + " ".join("%d:%d" % (x, c) for x, c in enumerate(cost)))


if __name__ == "__main__":
    main()
