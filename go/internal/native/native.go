// Package native is the cgo binding of the CUDA library (include/wva_b200.h).
//
// WRITTEN WITHOUT A GO TOOLCHAIN: the build image of this repository has no `go`, so this file has
// never been compiled.  It is the binding a maintainer drops into the reference tree (module
// github.com/llm-d-incubation/workload-variant-autoscaler) next to the replacement packages in
// go/pkg; build with CGO_ENABLED=1 (the reference Dockerfile:25 sets 0) and
//   CGO_CFLAGS=-I<repo>/include  CGO_LDFLAGS="-L<repo>/inferno-autoscaler_b200 -lwva_b200"
//
// cgo pointer rules (cmd/cgo "Passing pointers"):
//   (1) the library retains no Go pointer after a call returns (wva_b200.h "Conventions": it copies);
//   (2) a Go pointer passed to C must not point at memory that itself holds Go pointers.  The struct forms
//       wva_system_upload / wva_analyze_pairs / wva_solve take a struct OF pointers: a Go-allocated
//       C.wva_system_soa whose fields point at Go slices violates (2) and panics under the default
//       GODEBUG=cgocheck=1 ("cgo argument has Go pointer to unpinned Go pointer").  This binding therefore
//       calls the *_arrays forms of the header, where every slice is its own argument (a pointer to
//       pointer-free memory needs no pinning).  The only struct-of-pointers call is Group.Upload, which builds
//       the struct in C memory and pins every slice with runtime.Pinner for the duration of the call.
package native

/*
#cgo LDFLAGS: -lwva_b200
#include <stdlib.h>
#include "wva_b200.h"
*/
import "C"

import (
	"fmt"
	"runtime"
	"sync"
	"unsafe"
)

// SystemImage is the structure-of-arrays form of config.SystemSpec (wva_system_soa).
type SystemImage struct {
	S, A, M, T int

	AccCost         []float32
	AccMultiplicity []int32
	AccType         []int32
	TypeCapacity    []int64

	PerfAlpha, PerfBeta, PerfGamma, PerfDelta []float32
	PerfMaxBatch, PerfAtTokens, PerfAccCount  []int32
	PerfValid                                 []uint8

	SrvModel                         []int32
	SrvArrivalRPM                    []float32
	SrvInTokens, SrvOutTokens        []int32
	SrvSloTTFT, SrvSloITL, SrvSloTPS []float32
	SrvTargetValid                   []uint8
	SrvPriority, SrvMinReplicas      []int32
	SrvMaxBatch                      []int32
	SrvKeepAcc                       []uint8
	SrvCurAcc, SrvCurReplicas        []int32
	SrvCurCost                       []float32
}

// Allocs mirrors wva_alloc_soa (one record per index).
type Allocs struct {
	Acc                                   []int32
	NumReplicas, BatchSize                []int64
	Cost, Value, ITL, TTFT, Rho, MaxArrv []float32
}

func newAllocs(n int) *Allocs {
	return &Allocs{Acc: make([]int32, n), NumReplicas: make([]int64, n), BatchSize: make([]int64, n),
		Cost: make([]float32, n), Value: make([]float32, n), ITL: make([]float32, n), TTFT: make([]float32, n),
		Rho: make([]float32, n), MaxArrv: make([]float32, n)}
}

// Context wraps wva_ctx: one per process (creation builds the CUDA context), one call at a time —
// the same constraint the reference has through its package globals (pkg/core/system.go:12).
type Context struct {
	mu  sync.Mutex
	ctx *C.wva_ctx
}

var (
	defaultOnce sync.Once
	defaultCtx  *Context
	defaultErr  error
)

// Default returns the process-wide context on CUDA device 0 (WVA_B200_DEVICE overrides in the shim).
func Default() (*Context, error) {
	defaultOnce.Do(func() { defaultCtx, defaultErr = NewContext(0) })
	return defaultCtx, defaultErr
}

func NewContext(device int) (*Context, error) {
	var c *C.wva_ctx
	if rc := C.wva_ctx_create(C.int(device), &c); rc != C.WVA_OK {
		return nil, fmt.Errorf("wva_ctx_create: %d: %s", int(rc), C.GoString(C.wva_last_error(nil)))
	}
	ctx := &Context{ctx: c}
	runtime.SetFinalizer(ctx, func(x *Context) { C.wva_ctx_destroy(x.ctx) })
	return ctx, nil
}

func (c *Context) err(rc C.int, what string) error {
	if rc == C.WVA_OK {
		return nil
	}
	return fmt.Errorf("%s: %d: %s", what, int(rc), C.GoString(C.wva_last_error(c.ctx)))
}

func f32p(s []float32) *C.float { if len(s) == 0 { return nil }; return (*C.float)(unsafe.Pointer(&s[0])) }
func i32p(s []int32) *C.int32_t { if len(s) == 0 { return nil }; return (*C.int32_t)(unsafe.Pointer(&s[0])) }
func i64p(s []int64) *C.int64_t { if len(s) == 0 { return nil }; return (*C.int64_t)(unsafe.Pointer(&s[0])) }
func u8p(s []uint8) *C.uint8_t  { if len(s) == 0 { return nil }; return (*C.uint8_t)(unsafe.Pointer(&s[0])) }

// Upload replaces core.NewSystem + System.SetFromSpec on the native side (wva_system_upload).
func (c *Context) Upload(img *SystemImage) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	rc := C.wva_system_upload_arrays(c.ctx, C.int32_t(img.S), C.int32_t(img.A), C.int32_t(img.M), C.int32_t(img.T),
		f32p(img.AccCost), i32p(img.AccMultiplicity), i32p(img.AccType), i64p(img.TypeCapacity),
		f32p(img.PerfAlpha), f32p(img.PerfBeta), f32p(img.PerfGamma), f32p(img.PerfDelta),
		i32p(img.PerfMaxBatch), i32p(img.PerfAtTokens), i32p(img.PerfAccCount), u8p(img.PerfValid),
		i32p(img.SrvModel), f32p(img.SrvArrivalRPM), i32p(img.SrvInTokens), i32p(img.SrvOutTokens),
		f32p(img.SrvSloTTFT), f32p(img.SrvSloITL), f32p(img.SrvSloTPS), u8p(img.SrvTargetValid),
		i32p(img.SrvPriority), i32p(img.SrvMinReplicas), i32p(img.SrvMaxBatch), u8p(img.SrvKeepAcc),
		i32p(img.SrvCurAcc), i32p(img.SrvCurReplicas), f32p(img.SrvCurCost))
	return c.err(rc, "wva_system_upload_arrays")
}

// AnalyzePairs replaces Server.Calculate for all servers: S*A records + feasible flags.
func (c *Context) AnalyzePairs(s, a int) (*Allocs, []uint8, error) {
	c.mu.Lock()
	defer c.mu.Unlock()
	n := s * a
	if n == 0 {
		return newAllocs(0), nil, nil
	}
	out, fe := newAllocs(n), make([]uint8, n)
	rc := C.wva_analyze_pairs_arrays(c.ctx, i32p(out.Acc), i64p(out.NumReplicas), i64p(out.BatchSize), f32p(out.Cost), f32p(out.Value),
		f32p(out.ITL), f32p(out.TTFT), f32p(out.Rho), f32p(out.MaxArrv), u8p(fe))
	if err := c.err(rc, "wva_analyze_pairs_arrays"); err != nil {
		return nil, nil, err
	}
	return out, fe, nil
}

// Solve replaces solver.Solver.Solve: chosen candidate key per server (-1 = none) and a copy of it.
func (c *Context) Solve(s int, unlimited, delayedBestEffort bool, policy int) ([]int32, *Allocs, int64, error) {
	c.mu.Lock()
	defer c.mu.Unlock()
	b := func(v bool) C.int32_t { if v { return 1 }; return 0 }
	if s == 0 {
		return nil, newAllocs(0), 0, nil
	}
	key, out := make([]int32, s), newAllocs(s)
	rc := C.wva_solve_arrays(c.ctx, b(unlimited), b(delayedBestEffort), C.int32_t(policy), i32p(key),
		i32p(out.Acc), i64p(out.NumReplicas), i64p(out.BatchSize), f32p(out.Cost), f32p(out.Value),
		f32p(out.ITL), f32p(out.TTFT), f32p(out.Rho), f32p(out.MaxArrv))
	if err := c.err(rc, "wva_solve_arrays"); err != nil {
		return nil, nil, 0, err
	}
	return key, out, int64(C.wva_solution_time_usec(c.ctx)), nil
}

// AllocateByType replaces System.AllocateByType (per accelerator type totals of this process' shard).
func (c *Context) AllocateByType(t int) ([]int64, []float32, error) {
	c.mu.Lock()
	defer c.mu.Unlock()
	count, cost := make([]int64, t), make([]float32, t)
	if t == 0 {
		return count, cost, nil
	}
	return count, cost, c.err(C.wva_allocate_by_type(c.ctx, i64p(count), f32p(cost)), "wva_allocate_by_type")
}

// Analyze runs Server.Calculate for every pair of the shard and the candidate sweep side by side
// (wva_analyze); results stay on the device for Solve / PairsFetch / GridFetch.
func (c *Context) Analyze(rMax, bMax int) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	return c.err(C.wva_analyze(c.ctx, C.int32_t(rMax), C.int32_t(bMax), 0), "wva_analyze")
}

// Tuning knobs (results never depend on them; see include/wva_b200.h).  SolvePath: 2 = static-order scan (default),
// 1 = ranked queue, 0 = heap.  SweepFused: false = the sweep always stops at the host between its kernels.
func (c *Context) SetSolvePath(path int) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	return c.err(C.wva_solve_set_ranked(c.ctx, C.int32_t(path)), "wva_solve_set_ranked")
}

func (c *Context) SetSweepFused(on bool) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	v := C.int32_t(0)
	if on {
		v = 1
	}
	return c.err(C.wva_grid_set_fused(c.ctx, v), "wva_grid_set_fused")
}

// SetShard restricts the following calls to servers [first, first+count) (one process per GPU).
func (c *Context) SetShard(first, count int) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	return c.err(C.wva_set_shard(c.ctx, C.int32_t(first), C.int32_t(count)), "wva_set_shard")
}

// CommUniqueID / CommInit / CommShard: one process per GPU.  Rank 0 makes the 128-byte id, the caller
// distributes it (any transport), every rank attaches; from then on AllocateByType returns GLOBAL totals
// (the library runs the NCCL all-gather and the rank-order sum) and a limited Solve gathers the candidate
// rows itself.
func CommUniqueID() ([]byte, error) {
	id := make([]byte, C.WVA_COMM_ID_BYTES)
	if rc := C.wva_comm_unique_id(unsafe.Pointer(&id[0])); rc != C.WVA_OK {
		return nil, fmt.Errorf("wva_comm_unique_id: %d: %s", int(rc), C.GoString(C.wva_last_error(nil)))
	}
	return id, nil
}

func (c *Context) CommInit(id []byte, rank, nRanks int) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	if len(id) != C.WVA_COMM_ID_BYTES {
		return fmt.Errorf("communicator id must have %d bytes", int(C.WVA_COMM_ID_BYTES))
	}
	return c.err(C.wva_comm_init(c.ctx, unsafe.Pointer(&id[0]), C.int32_t(rank), C.int32_t(nRanks)), "wva_comm_init")
}

func (c *Context) CommShard() error {
	c.mu.Lock()
	defer c.mu.Unlock()
	return c.err(C.wva_comm_shard(c.ctx), "wva_comm_shard")
}

// TypeTotalsMerge sums the per-rank totals blocks that the host all-gathered (device memory,
// rank-major, 12*T bytes each) in rank order into this context's totals buffer: the exchange step of
// a sharded reconcile.  The collective itself belongs to the caller (NCCL / MPI binding of its choice).
func (c *Context) TypeTotalsMerge(gatheredDev unsafe.Pointer, nRanks int) error {
	c.mu.Lock()
	defer c.mu.Unlock()
	return c.err(C.wva_type_totals_merge(c.ctx, gatheredDev, C.int32_t(nRanks)), "wva_type_totals_merge")
}

// GridBest is wva_grid_best.
type GridBest struct {
	Acc, Replicas, Batch       int32
	Cost, Value, ITL, TTFT, Rho float32
}

// AnalyzeGrid runs the (server x accelerator x replicas x batch) candidate sweep; one winner per server.
func (c *Context) AnalyzeGrid(s, rMax, bMax int) ([]GridBest, error) {
	c.mu.Lock()
	defer c.mu.Unlock()
	best := make([]GridBest, s)
	if s == 0 {
		return best, nil
	}
	rc := C.wva_analyze_grid(c.ctx, C.int32_t(rMax), C.int32_t(bMax), (*C.wva_grid_best)(unsafe.Pointer(&best[0])), nil, nil)
	return best, c.err(rc, "wva_analyze_grid")
}

// GridBlocking returns the blocking probability p_block (float32 of the model's p[K], K = 11 b) of every candidate of
// the last successful sweep, indexed like the metric cube over the shard; NaN where Analyze does not accept the
// candidate.  The slice is sized by the library (wva_grid_blocking_size).  The plane also stays in HBM.
func (c *Context) GridBlocking() ([]float32, error) {
	c.mu.Lock()
	defer c.mu.Unlock()
	var n C.size_t
	if err := c.err(C.wva_grid_blocking_size(c.ctx, &n), "wva_grid_blocking_size"); err != nil {
		return nil, err
	}
	out := make([]float32, int(n))
	return out, c.err(C.wva_grid_blocking(c.ctx, f32p(out)), "wva_grid_blocking")
}

// GridBestBlocking returns p_block of each server's sweep winner (s servers of the shard), NaN where no candidate is
// feasible.  Needs neither the metric cube nor the plane of GridBlocking.
func (c *Context) GridBestBlocking(s int) ([]float32, error) {
	c.mu.Lock()
	defer c.mu.Unlock()
	out := make([]float32, s)
	if s == 0 {
		return out, nil
	}
	return out, c.err(C.wva_grid_best_blocking(c.ctx, f32p(out)), "wva_grid_best_blocking")
}

// PairRec is wva_pair_rec: one core.Allocation with its feasible flag, pointer-free (48 bytes, same layout as C).
type PairRec struct {
	Acc                    int32
	Feasible               uint8
	Pad                    [3]uint8
	NumReplicas, BatchSize int64
	Cost, Value, ITL, TTFT, Rho, MaxArrvRatePerReplica float32
}

func pairRecs(r []PairRec) *C.wva_pair_rec {
	if len(r) == 0 {
		return nil
	}
	return (*C.wva_pair_rec)(unsafe.Pointer(&r[0]))
}

// PairsAtBatchSizes sizes every pair of the shard under each ServerSpec.MaxBatchSize override of batches (strictly
// increasing, values in 1..8192): plane[((srv-first)*A+a)*len(batches)+j] is CreateAllocation's record under batches[j]
// (nil unless wantPlane), best[srv-first] is SolveUnlimited over the server's records.  The slices are sized from the
// library's own shard and dimensions.  The resident pair records, decisions and sweep results are left as they were.
func (c *Context) PairsAtBatchSizes(batches []int32, wantPlane bool) (plane, best []PairRec, err error) {
	c.mu.Lock()
	defer c.mu.Unlock()
	var S, A, M, T, first, count C.int32_t
	if err = c.err(C.wva_system_dims(c.ctx, &S, &A, &M, &T), "wva_system_dims"); err != nil {
		return nil, nil, err
	}
	if err = c.err(C.wva_shard_info(c.ctx, &first, &count), "wva_shard_info"); err != nil {
		return nil, nil, err
	}
	best = make([]PairRec, int(count))
	if wantPlane {
		plane = make([]PairRec, int(count)*int(A)*len(batches))
	}
	return plane, best, c.err(C.wva_analyze_pairs_batches(c.ctx, C.int32_t(len(batches)), i32p(batches), pairRecs(plane), pairRecs(best)),
		"wva_analyze_pairs_batches")
}

// PairsAtArrivalRates sizes every pair of the shard under each of nLoads arrival-rate scenarios: rpm[(srv-first)*nLoads+j]
// is the server's ServerLoadSpec.ArrivalRate (req/min) in scenario j.  plane[((srv-first)*nLoads+j)*A+a] is
// CreateAllocation's record of pair (srv, a) at that rate (nil unless wantPlane), best[(srv-first)*nLoads+j] is
// SolveUnlimited over those A records.  QueueAnalyzer.Size runs once per pair.  The slices are sized from the library's
// own shard and dimensions.  The resident image, pair records, decisions and sweep results are left as they were.
func (c *Context) PairsAtArrivalRates(rpm []float32, nLoads int, wantPlane bool) (plane, best []PairRec, err error) {
	c.mu.Lock()
	defer c.mu.Unlock()
	var S, A, M, T, first, count C.int32_t
	if err = c.err(C.wva_system_dims(c.ctx, &S, &A, &M, &T), "wva_system_dims"); err != nil {
		return nil, nil, err
	}
	if err = c.err(C.wva_shard_info(c.ctx, &first, &count), "wva_shard_info"); err != nil {
		return nil, nil, err
	}
	if nLoads < 1 || len(rpm) != int(count)*nLoads {
		return nil, nil, fmt.Errorf("PairsAtArrivalRates: rpm needs count*nLoads = %d*%d rates, got %d", int(count), nLoads, len(rpm))
	}
	best = make([]PairRec, int(count)*nLoads)
	if wantPlane {
		plane = make([]PairRec, int(count)*nLoads*int(A))
	}
	return plane, best, c.err(C.wva_analyze_pairs_loads(c.ctx, C.int32_t(nLoads), f32p(rpm), pairRecs(plane), pairRecs(best)),
		"wva_analyze_pairs_loads")
}

// CapacityScenarios is what SolveAtCapacities returns for nVec capacity vectors (and SolveAtArrivalRates for nLoads
// arrival-rate scenarios): Acc[j*S+s] and Chosen[j*S+s] are the limited solve's decision and chosen record (after
// best-effort scaling, Feasible = 1 where Acc >= 0) under vector (scenario) j,
// Count[j*T+t] and Cost[j*T+t] its AllocateByType totals over every server.
type CapacityScenarios struct {
	Acc    []int32
	Chosen []PairRec
	Count  []int64
	Cost   []float32
}

func solveCapacitiesArgs(S, T C.int32_t, capacity []int64, nVec int) (*CapacityScenarios, error) {
	if nVec < 1 || len(capacity) != nVec*int(T) {
		return nil, fmt.Errorf("SolveAtCapacities: capacity needs nVec*T = %d*%d counts, got %d", nVec, int(T), len(capacity))
	}
	return &CapacityScenarios{Acc: make([]int32, nVec*int(S)), Chosen: make([]PairRec, nVec*int(S)),
		Count: make([]int64, nVec*int(T)), Cost: make([]float32, nVec*int(T))}, nil
}

// SolveAtCapacities runs the limited solve once per capacity vector -- capacity[j*T .. j*T+T) is vector j, 1 <= nVec
// <= 8192 -- on the current pair records in one call: vector j gives what SetCapacity, a limited Solve and
// AllocateByType would.  The candidate order is built once; the pair records, the image's capacities and the last
// Solve's decisions are left as they were, so a later limited Solve needs no re-analysis.
func (c *Context) SolveAtCapacities(capacity []int64, nVec int, delayedBestEffort bool, policy int) (*CapacityScenarios, error) {
	c.mu.Lock()
	defer c.mu.Unlock()
	var S, A, M, T C.int32_t
	if err := c.err(C.wva_system_dims(c.ctx, &S, &A, &M, &T), "wva_system_dims"); err != nil {
		return nil, err
	}
	out, err := solveCapacitiesArgs(S, T, capacity, nVec)
	if err != nil {
		return nil, err
	}
	spec := C.wva_optimizer_spec{unlimited: 0, delayed_best_effort: 0, saturation_policy: C.int32_t(policy)}
	if delayedBestEffort {
		spec.delayed_best_effort = 1
	}
	return out, c.err(C.wva_solve_capacities(c.ctx, &spec, C.int32_t(nVec), i64p(capacity), i32p(out.Acc), pairRecs(out.Chosen),
		i64p(out.Count), f32p(out.Cost)), "wva_solve_capacities")
}

// SolveAtArrivalRates runs the limited solve once per arrival-rate scenario -- rpm[srv*nLoads+j] is server srv's
// ServerLoadSpec.ArrivalRate (req/min) in scenario j, 1 <= nLoads <= 8192, the layout of PairsAtArrivalRates -- under the
// image's capacities in one call: scenario j gives what UpdateServers with those rates, AnalyzePairs, a limited Solve and
// AllocateByType would, in CapacityScenarios' layout with j indexing scenarios.  QueueAnalyzer.Size runs once per pair
// and chunk.  The image, pair records and last Solve's decisions are left as they were; no AnalyzePairs is needed before
// it.  The context must hold every server (no shard).
func (c *Context) SolveAtArrivalRates(rpm []float32, nLoads int, delayedBestEffort bool, policy int) (*CapacityScenarios, error) {
	c.mu.Lock()
	defer c.mu.Unlock()
	var S, A, M, T C.int32_t
	if err := c.err(C.wva_system_dims(c.ctx, &S, &A, &M, &T), "wva_system_dims"); err != nil {
		return nil, err
	}
	if nLoads < 1 || len(rpm) != int(S)*nLoads {
		return nil, fmt.Errorf("SolveAtArrivalRates: rpm needs S*nLoads = %d*%d rates, got %d", int(S), nLoads, len(rpm))
	}
	out := &CapacityScenarios{Acc: make([]int32, nLoads*int(S)), Chosen: make([]PairRec, nLoads*int(S)),
		Count: make([]int64, nLoads*int(T)), Cost: make([]float32, nLoads*int(T))}
	spec := C.wva_optimizer_spec{unlimited: 0, delayed_best_effort: 0, saturation_policy: C.int32_t(policy)}
	if delayedBestEffort {
		spec.delayed_best_effort = 1
	}
	return out, c.err(C.wva_solve_loads(c.ctx, &spec, C.int32_t(nLoads), f32p(rpm), i32p(out.Acc), pairRecs(out.Chosen),
		i64p(out.Count), f32p(out.Cost)), "wva_solve_loads")
}

// QueueConfig is wva_queue_config; Metrics is wva_metrics (analyzer.AnalysisMetrics).
type QueueConfig struct {
	MaxBatchSize, MaxQueueSize int32
	Alpha, Beta, Gamma, Delta  float32
	AvgInputTokens, AvgOutputTokens int32
}
type Metrics struct {
	Throughput, AvgRespTime, AvgWaitTime, AvgNumInServ, AvgPrefillTime, AvgTokenTime, MaxRate, Rho float32
}

// QueueAnalyze: n independent QueueAnalyzer.Analyze calls.
func (c *Context) QueueAnalyze(cfg []QueueConfig, rate []float32) ([]Metrics, []uint8, error) {
	c.mu.Lock()
	defer c.mu.Unlock()
	n := len(cfg)
	m, st := make([]Metrics, n), make([]uint8, n)
	if n == 0 {
		return m, st, nil
	}
	rc := C.wva_queue_analyze(c.ctx, C.int32_t(n), (*C.wva_queue_config)(unsafe.Pointer(&cfg[0])), f32p(rate),
		(*C.wva_metrics)(unsafe.Pointer(&m[0])), u8p(st))
	return m, st, c.err(rc, "wva_queue_analyze")
}

// ModelSolve: a sequence of MM1ModelStateDependent.Solve(lambda[i], mu[i]) calls on one model
// NewMM1ModelStateDependent(K, servRate); out has 9 floats per call {isValid, rho, avgRespTime, avgWaitTime,
// avgServTime, avgNumInSystem, avgQueueLength, avgNumInServers, throughput}; p = probabilities after the last call.
func (c *Context) ModelSolve(K int, servRate, lambda, mu []float32) (out []float32, p []float64, err error) {
	c.mu.Lock()
	defer c.mu.Unlock()
	n := len(lambda)
	out, p = make([]float32, 9*n), make([]float64, K+1)
	if n == 0 || len(servRate) == 0 || len(mu) != n {
		return out, p, fmt.Errorf("bad ModelSolve arguments")
	}
	rc := C.wva_model_solve(c.ctx, C.int64_t(K), f32p(servRate), C.int32_t(len(servRate)), C.int32_t(n), f32p(lambda), f32p(mu),
		f32p(out), (*C.double)(unsafe.Pointer(&p[0])))
	return out, p, c.err(rc, "wva_model_solve")
}

// QueueSize: n independent QueueAnalyzer.Size calls; target/rates/achieved are (TTFT, ITL, TPS) triples.
func (c *Context) QueueSize(cfg []QueueConfig, target []float32) (rates []float32, m []Metrics, achieved []float32, status []uint8, err error) {
	c.mu.Lock()
	defer c.mu.Unlock()
	n := len(cfg)
	rates, achieved, m, status = make([]float32, 3*n), make([]float32, 3*n), make([]Metrics, n), make([]uint8, n)
	if n == 0 {
		return
	}
	rc := C.wva_queue_size(c.ctx, C.int32_t(n), (*C.wva_queue_config)(unsafe.Pointer(&cfg[0])), f32p(target), f32p(rates),
		(*C.wva_metrics)(unsafe.Pointer(&m[0])), f32p(achieved), u8p(status))
	err = c.err(rc, "wva_queue_size")
	return
}

// Group wraps wva_group: ONE process (the single reconcile goroutine of
// internal/controller/variantautoscaling_controller.go:143-166) driving every GPU of the box.  Servers are
// sharded over the devices by the library; outputs have the full extent; totals are global.
type Group struct {
	mu sync.Mutex
	g  *C.wva_group
	n  int
}

func NewGroup(devices []int32) (*Group, error) {
	if len(devices) == 0 {
		return nil, fmt.Errorf("no devices")
	}
	var g *C.wva_group
	if rc := C.wva_group_create(i32p(devices), C.int32_t(len(devices)), &g); rc != C.WVA_OK {
		return nil, fmt.Errorf("wva_group_create: %d: %s", int(rc), C.GoString(C.wva_last_error(nil)))
	}
	grp := &Group{g: g, n: len(devices)}
	runtime.SetFinalizer(grp, func(x *Group) { C.wva_group_destroy(x.g) })
	return grp, nil
}

func (g *Group) err(rc C.int, what string) error {
	if rc == C.WVA_OK {
		return nil
	}
	return fmt.Errorf("%s: %d: %s", what, int(rc), C.GoString(C.wva_group_last_error(g.g)))
}

// Upload replicates the image on every device and shards the servers.  wva_group_upload takes the struct
// form, so the slices are pinned for the duration of the call (runtime.Pinner, Go >= 1.21; the reference
// is on go1.23, go.mod:7) -- the one place this binding builds a C struct of Go pointers.
func (g *Group) Upload(img *SystemImage) error {
	g.mu.Lock()
	defer g.mu.Unlock()
	var pin runtime.Pinner
	defer pin.Unpin()
	pf := func(s []float32) *C.float { if len(s) == 0 { return nil }; pin.Pin(&s[0]); return (*C.float)(unsafe.Pointer(&s[0])) }
	pi := func(s []int32) *C.int32_t { if len(s) == 0 { return nil }; pin.Pin(&s[0]); return (*C.int32_t)(unsafe.Pointer(&s[0])) }
	pl := func(s []int64) *C.int64_t { if len(s) == 0 { return nil }; pin.Pin(&s[0]); return (*C.int64_t)(unsafe.Pointer(&s[0])) }
	pu := func(s []uint8) *C.uint8_t { if len(s) == 0 { return nil }; pin.Pin(&s[0]); return (*C.uint8_t)(unsafe.Pointer(&s[0])) }
	h := (*C.wva_system_soa)(C.calloc(1, C.size_t(unsafe.Sizeof(C.wva_system_soa{}))))   // C memory: may hold pinned Go pointers
	defer C.free(unsafe.Pointer(h))
	h.n_servers, h.n_accels, h.n_models, h.n_types = C.int32_t(img.S), C.int32_t(img.A), C.int32_t(img.M), C.int32_t(img.T)
	h.acc_cost, h.acc_multiplicity, h.acc_type, h.type_capacity = pf(img.AccCost), pi(img.AccMultiplicity), pi(img.AccType), pl(img.TypeCapacity)
	h.perf_alpha, h.perf_beta, h.perf_gamma, h.perf_delta = pf(img.PerfAlpha), pf(img.PerfBeta), pf(img.PerfGamma), pf(img.PerfDelta)
	h.perf_max_batch, h.perf_at_tokens, h.perf_acc_count, h.perf_valid = pi(img.PerfMaxBatch), pi(img.PerfAtTokens), pi(img.PerfAccCount), pu(img.PerfValid)
	h.srv_model, h.srv_arrival_rpm, h.srv_in_tokens, h.srv_out_tokens = pi(img.SrvModel), pf(img.SrvArrivalRPM), pi(img.SrvInTokens), pi(img.SrvOutTokens)
	h.srv_slo_ttft, h.srv_slo_itl, h.srv_slo_tps, h.srv_target_valid = pf(img.SrvSloTTFT), pf(img.SrvSloITL), pf(img.SrvSloTPS), pu(img.SrvTargetValid)
	h.srv_priority, h.srv_min_replicas, h.srv_max_batch, h.srv_keep_acc = pi(img.SrvPriority), pi(img.SrvMinReplicas), pi(img.SrvMaxBatch), pu(img.SrvKeepAcc)
	h.srv_cur_acc, h.srv_cur_replicas, h.srv_cur_cost = pi(img.SrvCurAcc), pi(img.SrvCurReplicas), pf(img.SrvCurCost)
	return g.err(C.wva_group_upload(g.g, h), "wva_group_upload")
}

// Analyze: Server.Calculate for every pair (and the candidate sweep when rMax > 0) on all devices.
func (g *Group) Analyze(rMax, bMax int) error {
	g.mu.Lock()
	defer g.mu.Unlock()
	return g.err(C.wva_group_analyze(g.g, C.int32_t(rMax), C.int32_t(bMax), 0), "wva_group_analyze")
}

// GridBestBlocking: p_block of every server's sweep winner (s servers), assembled from the devices' shards.
func (g *Group) GridBestBlocking(s int) ([]float32, error) {
	g.mu.Lock()
	defer g.mu.Unlock()
	out := make([]float32, s)
	if s == 0 {
		return out, nil
	}
	return out, g.err(C.wva_group_grid_best_blocking(g.g, f32p(out)), "wva_group_grid_best_blocking")
}

// PairsAtBatchSizes: Context.PairsAtBatchSizes over every device's servers, assembled (sized from device 0's image).
func (g *Group) PairsAtBatchSizes(batches []int32, wantPlane bool) (plane, best []PairRec, err error) {
	g.mu.Lock()
	defer g.mu.Unlock()
	var S, A, M, T C.int32_t
	if rc := C.wva_system_dims(C.wva_group_ctx(g.g, 0), &S, &A, &M, &T); rc != C.WVA_OK {
		return nil, nil, fmt.Errorf("wva_system_dims: %d", int(rc))
	}
	best = make([]PairRec, int(S))
	if wantPlane {
		plane = make([]PairRec, int(S)*int(A)*len(batches))
	}
	return plane, best, g.err(C.wva_group_analyze_pairs_batches(g.g, C.int32_t(len(batches)), i32p(batches), pairRecs(plane), pairRecs(best)),
		"wva_group_analyze_pairs_batches")
}

// PairsAtArrivalRates: Context.PairsAtArrivalRates over every device's servers, assembled: rpm holds S*nLoads rates
// (sized from device 0's image).
func (g *Group) PairsAtArrivalRates(rpm []float32, nLoads int, wantPlane bool) (plane, best []PairRec, err error) {
	g.mu.Lock()
	defer g.mu.Unlock()
	var S, A, M, T C.int32_t
	if rc := C.wva_system_dims(C.wva_group_ctx(g.g, 0), &S, &A, &M, &T); rc != C.WVA_OK {
		return nil, nil, fmt.Errorf("wva_system_dims: %d", int(rc))
	}
	if nLoads < 1 || len(rpm) != int(S)*nLoads {
		return nil, nil, fmt.Errorf("PairsAtArrivalRates: rpm needs S*nLoads = %d*%d rates, got %d", int(S), nLoads, len(rpm))
	}
	best = make([]PairRec, int(S)*nLoads)
	if wantPlane {
		plane = make([]PairRec, int(S)*nLoads*int(A))
	}
	return plane, best, g.err(C.wva_group_analyze_pairs_loads(g.g, C.int32_t(nLoads), f32p(rpm), pairRecs(plane), pairRecs(best)),
		"wva_group_analyze_pairs_loads")
}

// SolveAtCapacities: Context.SolveAtCapacities on every device's gathered rows; device 0 returns the results.
func (g *Group) SolveAtCapacities(capacity []int64, nVec int, delayedBestEffort bool, policy int) (*CapacityScenarios, error) {
	g.mu.Lock()
	defer g.mu.Unlock()
	var S, A, M, T C.int32_t
	if rc := C.wva_system_dims(C.wva_group_ctx(g.g, 0), &S, &A, &M, &T); rc != C.WVA_OK {
		return nil, fmt.Errorf("wva_system_dims: %d", int(rc))
	}
	out, err := solveCapacitiesArgs(S, T, capacity, nVec)
	if err != nil {
		return nil, err
	}
	spec := C.wva_optimizer_spec{unlimited: 0, delayed_best_effort: 0, saturation_policy: C.int32_t(policy)}
	if delayedBestEffort {
		spec.delayed_best_effort = 1
	}
	return out, g.err(C.wva_group_solve_capacities(g.g, &spec, C.int32_t(nVec), i64p(capacity), i32p(out.Acc), pairRecs(out.Chosen),
		i64p(out.Count), f32p(out.Cost)), "wva_group_solve_capacities")
}

// AllocateByType: global per-type totals (NCCL all-gather of the partials inside the library).
func (g *Group) AllocateByType(t int) ([]int64, []float32, error) {
	g.mu.Lock()
	defer g.mu.Unlock()
	count, cost := make([]int64, t), make([]float32, t)
	if t == 0 {
		return count, cost, nil
	}
	return count, cost, g.err(C.wva_group_allocate_by_type(g.g, i64p(count), f32p(cost)), "wva_group_allocate_by_type")
}
