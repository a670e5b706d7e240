// Package solver — drop-in replacement of the reference's pkg/solver (optimizer.go, solver.go,
// greedy.go): same exported identifiers; SolveUnlimited / SolveGreedy run in the CUDA library.
// WRITTEN WITHOUT A GO TOOLCHAIN; never compiled (INTEGRATION.md).
package solver

import (
	"fmt"

	"github.com/llm-d-incubation/workload-variant-autoscaler/go/internal/native"
	"github.com/llm-d-incubation/workload-variant-autoscaler/go/pkg/core"
	"github.com/llm-d-incubation/workload-variant-autoscaler/pkg/config"
)

type Solver struct {
	optimizerSpec     *config.OptimizerSpec
	currentAllocation map[string]*core.Allocation
	diffAllocation    map[string]*core.AllocationDiff
	solutionTimeUsec  int64
}

func NewSolver(spec *config.OptimizerSpec) *Solver {
	return &Solver{optimizerSpec: spec, currentAllocation: map[string]*core.Allocation{}, diffAllocation: map[string]*core.AllocationDiff{}}
}

// Solve (solver.go:32-60)
func (s *Solver) Solve() error {
	s.currentAllocation = map[string]*core.Allocation{}
	for name, server := range core.GetServers() {
		if a := server.CurAllocation(); a != nil {
			s.currentAllocation[name] = a
		}
	}
	usec, err := core.TheSystem.Solve(s.optimizerSpec)
	if err != nil {
		return err
	}
	s.solutionTimeUsec = usec
	// solver.go:46-57: diff of current vs desired allocation per server
	s.diffAllocation = map[string]*core.AllocationDiff{}
	for name, server := range core.GetServers() {
		if d := core.CreateAllocationDiff(s.currentAllocation[name], server.Allocation()); d != nil {
			s.diffAllocation[name] = d
		}
	}
	return nil
}

// SolveUnlimited / SolveGreedy keep the reference's entry points (solver.go:63, greedy.go:35).
func (s *Solver) SolveUnlimited() { spec := *s.optimizerSpec; spec.Unlimited = true; _, _ = core.TheSystem.Solve(&spec) }
func (s *Solver) SolveGreedy()    { spec := *s.optimizerSpec; spec.Unlimited = false; _, _ = core.TheSystem.Solve(&spec) }
// AllocationDiff (solver.go:81): the reference's return type.
func (s *Solver) AllocationDiff() map[string]*core.AllocationDiff { return s.diffAllocation }

// SolveAtCapacities answers "what would SolveGreedy decide under these capacities?" for nVec capacity vectors at once
// (capacity[j*T+t]: vector j, accelerator type t of the system) without changing the system's allocations or capacities.
func (s *Solver) SolveAtCapacities(capacity []int64, nVec int) (*native.CapacityScenarios, error) {
	spec := *s.optimizerSpec
	spec.Unlimited = false
	return core.TheSystem.SolveAtCapacities(&spec, capacity, nVec)
}

// SolveAtArrivalRates answers "what would SolveGreedy decide at these loads?" for nLoads arrival-rate scenarios at once
// (rpm[srv*nLoads+j]: server srv's ArrivalRate in req/min in scenario j) on the system's capacities, without changing
// the system's allocations, loads or capacities.
func (s *Solver) SolveAtArrivalRates(rpm []float32, nLoads int) (*native.CapacityScenarios, error) {
	spec := *s.optimizerSpec
	spec.Unlimited = false
	return core.TheSystem.SolveAtArrivalRates(&spec, rpm, nLoads)
}

type Optimizer struct {
	spec             *config.OptimizerSpec
	solver           *Solver
	solutionTimeMsec int64
}

func NewOptimizerFromSpec(spec *config.OptimizerSpec) *Optimizer { return &Optimizer{spec: spec} }

// Optimize (optimizer.go:24-35); SolutionTimeMsec is the device+host time of the native solve.
func (o *Optimizer) Optimize() error {
	if o.spec == nil {
		return fmt.Errorf("missing optimizer spec")
	}
	o.solver = NewSolver(o.spec)
	err := o.solver.Solve()
	o.solutionTimeMsec = o.solver.solutionTimeUsec / 1000
	return err
}
func (o *Optimizer) SolutionTimeMsec() int64 { return o.solutionTimeMsec }
