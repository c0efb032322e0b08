"""Prompt prefix cache policy: which pool block holds the KV rows of which token block (pure host code, no torch).

The reference's PrefixCache (src/generator/prefix_cache.hpp:35-117) keys a block by its own tokens and its index, so
after [A, B] and [C, B] a prompt [C, B, ...] would load the B rows computed after A.  Here the blocks form a trie: a
block's key is (its parent block, its tokens), so a block stands for the whole prefix up to its end and identical token
runs after different prefixes never match.

Every decision depends only on the sequence of calls.  Each tensor-parallel rank keeps its own pool of its own KV heads
and its own PrefixCache; given the same calls they pick the same blocks with no exchange.
"""
from collections import OrderedDict


class _Node:
    __slots__ = ("parent", "tokens", "block", "children")

    def __init__(self, parent, tokens, block):
        self.parent = parent
        self.tokens = tokens
        self.block = block
        self.children = {}


class PrefixCache:
    def __init__(self, num_blocks, block_tokens):
        if num_blocks <= 0 or block_tokens <= 0:
            raise ValueError("num_blocks and block_tokens must be positive")
        self.num_blocks = int(num_blocks)
        self.block_tokens = int(block_tokens)
        self._root = _Node(None, (), -1)
        self._free = list(range(self.num_blocks - 1, -1, -1))   # pop() hands out block 0 first
        self._lru = OrderedDict()                                # cached node -> None, least recently used first

    def _blocks(self, tokens):
        """token blocks of a prompt that may come from the cache: at most (len - 1) // bt, so that at least one token is
        always prefilled and yields the next-token logits"""
        bt = self.block_tokens
        toks = [int(t) for t in tokens]
        return [tuple(toks[j * bt:(j + 1) * bt]) for j in range((len(toks) - 1) // bt if toks else 0)]

    def _touch(self, nodes):
        for nd in nodes:   # parents first: a child is always more recent than its parent
            self._lru.move_to_end(nd)

    def _walk(self, blocks):
        path, nd = [], self._root
        for key in blocks:
            nd = nd.children.get(key)
            if nd is None:
                break
            path.append(nd)
        return path

    def match(self, tokens):
        """-> pool blocks of the longest cached prefix of `tokens`, in task-block order (block j holds rows
        [j bt, (j + 1) bt)).  Refreshes their LRU position."""
        path = self._walk(self._blocks(tokens))
        self._touch(path)
        return [nd.block for nd in path]

    def _evict(self, keep):
        """the least recently used cached block without cached children, not in `keep`; None when there is none"""
        for nd in self._lru:
            if not nd.children and nd not in keep:
                del self._lru[nd]
                del nd.parent.children[nd.tokens]
                return nd.block
        return None

    def insert(self, tokens):
        """Cache the blocks of `tokens` that match() could serve and are not cached yet.  -> [(task block, pool block)]
        to save from the task that holds the prompt's rows.  Free blocks go first, then least recently used blocks
        without cached children; a block is never evicted while it has cached children, nor while it is on this
        prompt's path.  Stops early when no block can be had."""
        blocks = self._blocks(tokens)
        path = self._walk(blocks)
        self._touch(path)
        keep = set(path)
        parent = path[-1] if path else self._root
        out = []
        for j in range(len(path), len(blocks)):
            pb = self._free.pop() if self._free else self._evict(keep)
            if pb is None:
                break
            nd = _Node(parent, blocks[j], pb)
            parent.children[blocks[j]] = nd
            self._lru[nd] = None
            keep.add(nd)
            out.append((j, pb))
            parent = nd
        return out

    def __len__(self):
        return len(self._lru)
