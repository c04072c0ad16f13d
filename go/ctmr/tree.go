// cgo binding of the Merkle tree forms of include/ctmr_frontend.h: the entries a run ingests, folded into the log's
// RFC 6962 Merkle tree on the GPU, so that the run can be checked against the log's signed tree head.
//
// NOT COMPILED IN THIS REPOSITORY'S CI: the build image has no Go toolchain.  See INTEGRATION.md §2b and §2c.
package ctmr

/*
#include "ctmr_frontend.h"
*/
import "C"

import "unsafe"

// Tree mirrors ctmr_tree: the Merkle tree over the first Size entries of one log, held as its right edge.  It holds no
// pointers, so it is passed to the library straight from Go memory.  Keep it next to LogState: a restarted run resumes
// the tree from it.
type Tree struct {
	Size uint64
	Edge [64][32]byte // for every bit k set in Size, the root of the complete subtree of 2^k leaves ending below Size
	Root [32]byte     // MTH of the first Size entries after the call; compare with SHA256RootHash / the checkpoint
}

// the layouts agree, or this does not compile
var _ [unsafe.Sizeof(C.ctmr_tree{}) - unsafe.Sizeof(Tree{})]struct{}
var _ [unsafe.Sizeof(Tree{}) - unsafe.Sizeof(C.ctmr_tree{})]struct{}

func (t *Tree) c() *C.ctmr_tree { return (*C.ctmr_tree)(unsafe.Pointer(t)) }

// NoTree mirrors CTMR_NO_TREE: an entry or tile that folds into no tree.  MaxTrees mirrors CTMR_MAX_TREES.
const (
	NoTree   = uint32(C.CTMR_NO_TREE)
	MaxTrees = int(C.CTMR_MAX_TREES)
)

// treesC passes a []Tree to the library straight from Go memory: Tree holds no pointers.
func treesC(trees []Tree) *C.ctmr_tree {
	if len(trees) == 0 {
		return nil
	}
	return trees[0].c()
}

// ProcessRawTree is ProcessRaw, and the pages' entries folded into tree as the log's entries tree.Size, tree.Size+1, ....
// An entry whose leaf_input is not base64 has no leaf: the fold stops before it and tree.Size says where.  On an error
// tree is unchanged.  On a group the GPUs fold their chunks in log order and the tree is the one-GPU tree.
func (d *DB) ProcessRawTree(p *RawPages, nowUnixNs int64, r *RawResult, tree *Tree) error {
	return d.processRaw(p, nowUnixNs, r, tree, nil, false)
}

// ProcessRawTrees is ProcessRaw, and every entry folded into the tree of its log: the entries of a body added with
// AppendLog(body, log) are the next leaves of trees[log]; those added with Append fold nowhere.  This is the one flush
// of a batcher that drains the pages of every log it syncs into one RawPages: each log keeps the one-tree rules on its
// own entries, and a bad base64 leaf_input stops only its own log's tree.  Every tree gets its root written, also a tree
// with no entry in the batch.  On an error every tree is unchanged.  On one GPU or a group.
func (d *DB) ProcessRawTrees(p *RawPages, nowUnixNs int64, r *RawResult, trees []Tree) error {
	return d.processRaw(p, nowUnixNs, r, nil, trees, true)
}

// ProcessRawBodiesTree is ProcessRawBodies, and the bodies' entries folded into tree: entry j of a body recorded with
// CommitLog / AppendBodyLog(..., start, log) is the log's entry start + j.  The bodies are walked in the order recorded
// from tree.Size on: entries below it are already in the tree and are skipped, a body whose status is not BodyOK or that
// starts above it (a short answer left a gap) stops the fold, and so does the first entry whose leaf_input is not
// base64.  A stop is final for the call: fetch again from tree.Size.  A BodyRepeatedEntries body stops the fold too: its
// entries still go through ProcessRaw, decoded on the host, but without a tree, so fetch that range again and fold it
// with the next call.  The starts must not decrease and the first must not lie above tree.Size (CTMR_E_INVALID before
// any work, tree unchanged).  Every output is that of ProcessRawBodies.  On one GPU or a group.
func (d *DB) ProcessRawBodiesTree(p *RawBodies, nowUnixNs int64, r *BodiesResult, fallback *RawPages,
	newResult func(n int) *RawResult, tree *Tree) (*Repeated, error) {
	return d.processRawBodies(p, nowUnixNs, r, fallback, newResult, tree, nil, false)
}

// ProcessRawBodiesTrees is ProcessRawBodiesTree for the bodies of many logs in one batch: the entries of a body recorded
// with CommitLog / AppendBodyLog(..., start, log) fold into trees[log], each log's bodies with the one-tree rules on their
// own; bodies of Commit / AppendBody fold nowhere.  Every tree gets its root written.  On an error every tree is
// unchanged.  On one GPU or a group.
func (d *DB) ProcessRawBodiesTrees(p *RawBodies, nowUnixNs int64, r *BodiesResult, fallback *RawPages,
	newResult func(n int) *RawResult, trees []Tree) (*Repeated, error) {
	return d.processRawBodies(p, nowUnixNs, r, fallback, newResult, nil, trees, true)
}

// ProcessTilesTree is ProcessTiles, and the tiles' entries folded into tree.  The tiles must be consecutive tiles of one
// log, full but for the last, with tree.Size inside the first: its leaves below tree.Size are skipped.  A bad tile stops
// the fold at its first leaf, and the rest of the batch is still processed.  The fetch/register/resume loop carries the
// tree from call to call; once a bad tile has stopped the fold, it resumes with ProcessTiles' plain call and the tree
// stays as it is.  Tree and outputs equal those of one call with every certificate registered first.  On one GPU or a
// group.
func (d *DB) ProcessTilesTree(t *Tiles, nowUnixNs int64, r *TileResult, fetch func(fp [32]byte) ([]byte, error), tree *Tree) error {
	return d.processTiles(t, nowUnixNs, r, fetch, tree, nil, false)
}

// ProcessTilesTrees is ProcessTiles, and every tile folded into the tree of its log: a tile added with
// AppendLog(body, index, width, log) is the next tile of trees[log]; one added with Append folds nowhere.  Each log's
// tiles keep ProcessTilesTree's rules in batch order, interleaved with the other logs' in any way.  The resume loop
// carries the trees; a log whose tree a bad tile stopped (its size is below its first remaining tile) goes on as
// NoTree.  Trees and outputs equal those of one call with every certificate registered first.  On one GPU or a group.
func (d *DB) ProcessTilesTrees(t *Tiles, nowUnixNs int64, r *TileResult, fetch func(fp [32]byte) ([]byte, error), trees []Tree) error {
	return d.processTiles(t, nowUnixNs, r, fetch, nil, trees, true)
}
