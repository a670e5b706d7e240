// Package core — drop-in replacement of the reference's pkg/core for the Analyze -> Optimize path.
//
// Same exported identifiers as the reference (pkg/core/system.go, server.go, allocation.go,
// accelerator.go, model.go, serviceclass.go); the arithmetic of CreateAllocation / Server.Calculate /
// AllocateByType runs in the CUDA library through go/internal/native.  pkg/config is the reference's
// own package (plain data) and is imported unchanged.
//
// WRITTEN WITHOUT A GO TOOLCHAIN (none in the build image): never compiled; see INTEGRATION.md.
//
// Behavioural notes
//   - Server.Calculate sizes EVERY server of the System in one native call the first time it is invoked
//     after SetFromSpec, then serves each server from that result.  The reference's AnalyzeModel also
//     works by side effect on the shared System (internal/modelanalyzer/analyzer.go:29-31), and
//     Optimize ignores its `analysis` argument (internal/optimizer/optimizer.go:30-54), so the
//     controller cannot observe the difference.
//   - Go map iteration order is random in the reference; the native side fixes it to dense-index order
//     (ties only).
package core

import (
	"fmt"

	"github.com/llm-d-incubation/workload-variant-autoscaler/go/internal/native"
	"github.com/llm-d-incubation/workload-variant-autoscaler/pkg/config"
)

// TheSystem: the reference keeps a package-level singleton (system.go:12); manager.NewManager sets it.
var TheSystem *System

func GetServers() map[string]*Server            { return TheSystem.servers }
func GetServer(name string) *Server             { return TheSystem.servers[name] }
func GetAccelerators() map[string]*Accelerator  { return TheSystem.accelerators }
func GetAccelerator(name string) *Accelerator   { return TheSystem.accelerators[name] }
func GetModels() map[string]*Model              { return TheSystem.models }
func GetModel(name string) *Model               { return TheSystem.models[name] }
func GetServiceClass(name string) *ServiceClass { return TheSystem.serviceClasses[name] }
func GetCapacities() map[string]int             { return TheSystem.capacity }

// ---- plain data holders (accelerator.go, model.go, serviceclass.go) -----------------------------

type Accelerator struct {
	name string
	spec *config.AcceleratorSpec
}

func NewAcceleratorFromSpec(spec *config.AcceleratorSpec) *Accelerator { return &Accelerator{name: spec.Name, spec: spec} }
func (g *Accelerator) Name() string                  { return g.name }
func (g *Accelerator) Spec() *config.AcceleratorSpec { return g.spec }
func (g *Accelerator) Type() string                  { return g.spec.Type }
func (g *Accelerator) Cost() float32                 { return g.spec.Cost }
func (g *Accelerator) Multiplicity() int             { return g.spec.Multiplicity }
func (g *Accelerator) MemSize() int                  { return g.spec.MemSize }
func (g *Accelerator) Calculate()                    {}

type Model struct {
	name         string
	perfData     map[string]*config.ModelAcceleratorPerfData
	numInstances map[string]int
}

func NewModel(name string) *Model {
	return &Model{name: name, perfData: map[string]*config.ModelAcceleratorPerfData{}, numInstances: map[string]int{}}
}
func (m *Model) Name() string                                        { return m.name }
func (m *Model) NumInstances(acc string) int                         { return m.numInstances[acc] }
func (m *Model) PerfData(acc string) *config.ModelAcceleratorPerfData { return m.perfData[acc] }
func (m *Model) Calculate(map[string]*Accelerator)                   {}
func (m *Model) AddPerfDataFromSpec(spec *config.ModelAcceleratorPerfData) {
	if spec.Name != m.name {
		return
	}
	m.perfData[spec.Acc] = spec
	count := spec.AccCount
	if count <= 0 {
		count = 1
	}
	m.numInstances[spec.Acc] = count
}

type Target struct{ ITL, TTFT, TPS float32 }

type ServiceClass struct {
	name     string
	priority int
	targets  map[string]*Target
}

func NewServiceClass(name string, priority int) *ServiceClass {
	if priority < config.DefaultHighPriority || priority > config.DefaultLowPriority {
		priority = config.DefaultServiceClassPriority
	}
	return &ServiceClass{name: name, priority: priority, targets: map[string]*Target{}}
}
func NewServiceClassFromSpec(spec *config.ServiceClassSpec) *ServiceClass {
	svc := NewServiceClass(spec.Name, spec.Priority)
	for i := range spec.ModelTargets {
		svc.AddModelTarget(&spec.ModelTargets[i])
	}
	return svc
}
func (c *ServiceClass) Name() string                  { return c.name }
func (c *ServiceClass) Priority() int                 { return c.priority }
func (c *ServiceClass) ModelTarget(m string) *Target  { return c.targets[m] }
func (c *ServiceClass) AddModelTarget(spec *config.ModelTarget) *Target {
	t := &Target{ITL: spec.SLO_ITL, TTFT: spec.SLO_TTFT, TPS: spec.SLO_TPS}
	c.targets[spec.Model] = t
	return t
}

// ---- Allocation (allocation.go:13-24 and its accessors) ------------------------------------------

type Allocation struct {
	accelerator           string
	numReplicas           int
	batchSize             int
	cost, value           float32
	itl, ttft, rho        float32
	maxArrvRatePerReplica float32
}

func (a *Allocation) Accelerator() string            { return a.accelerator }
func (a *Allocation) NumReplicas() int               { return a.numReplicas }
func (a *Allocation) SetNumReplicas(n int)           { a.numReplicas = n }
func (a *Allocation) MaxBatchSize() int              { return a.batchSize }
func (a *Allocation) SetMaxBatchSize(b int)          { a.batchSize = b }
func (a *Allocation) MaxArrvRatePerReplica() float32 { return a.maxArrvRatePerReplica }
func (a *Allocation) MaxRPM() float32                { return a.maxArrvRatePerReplica * 1000 * 60 }
func (a *Allocation) Cost() float32                  { return a.cost }
func (a *Allocation) SetCost(c float32)              { a.cost = c }
func (a *Allocation) Value() float32                 { return a.value }
func (a *Allocation) SetValue(v float32)             { a.value = v }
func (a *Allocation) Saturated(totalRate float32) bool {
	return totalRate > float32(a.numReplicas)*a.MaxRPM()
}
func (a *Allocation) Clone() *Allocation { c := *a; return &c }
func (a *Allocation) AllocationData() *config.AllocationData {
	return &config.AllocationData{Accelerator: a.accelerator, NumReplicas: a.numReplicas, MaxBatch: a.batchSize,
		Cost: a.cost, ITLAverage: a.itl, TTFTAverage: a.ttft}
}
func AllocationFromData(d *config.AllocationData) *Allocation {
	return &Allocation{accelerator: d.Accelerator, numReplicas: d.NumReplicas, batchSize: d.MaxBatch, cost: d.Cost,
		itl: d.ITLAverage, ttft: d.TTFTAverage}
}
func (a *Allocation) String() string {
	return fmt.Sprintf("{acc=%s; numRep=%d; maxBatch=%d; cost=%v, val=%v, itl=%v, ttft=%v, rho=%v, maxRPM=%v}",
		a.accelerator, a.numReplicas, a.batchSize, a.cost, a.value, a.itl, a.ttft, a.rho, a.MaxRPM())
}

// CreateAllocation keeps the reference's entry point (allocation.go:27): the record the native sweep
// produced for (server, accelerator), value = cost as in the reference (Server.Calculate then stores
// the transition penalty).  nil when infeasible.
func CreateAllocation(serverName string, gName string) *Allocation {
	s := TheSystem
	if s == nil {
		return nil
	}
	if err := s.analyzeAll(); err != nil {
		return nil
	}
	si, ok := s.serverIndex[serverName]
	ai, ok2 := s.accIndex[gName]
	if !ok || !ok2 {
		return nil
	}
	al := s.pairAllocation(si, ai, true)
	if al != nil {
		al.value = al.cost
	}
	return al
}

// ---- Server (server.go) ---------------------------------------------------------------------------

type Server struct {
	name, serviceClassName, modelName string
	keepAccelerator                   bool
	minNumReplicas, maxBatchSize      int
	load                              *config.ServerLoadSpec
	allAllocations                    map[string]*Allocation
	allocation, curAllocation         *Allocation
	spec                              *config.ServerSpec
	system                            *System
	index                             int
}

func NewServerFromSpec(spec *config.ServerSpec) *Server {
	ld := spec.CurrentAlloc.Load
	svc := spec.Class
	if svc == "" {
		svc = config.DefaultServiceClassName
	}
	return &Server{name: spec.Name, serviceClassName: svc, modelName: spec.Model, load: &ld,
		keepAccelerator: spec.KeepAccelerator, minNumReplicas: spec.MinNumReplicas, maxBatchSize: spec.MaxBatchSize,
		allAllocations: map[string]*Allocation{}, curAllocation: AllocationFromData(&spec.CurrentAlloc), spec: spec}
}

// Calculate (server.go:55-67).  The `accelerators` argument is the System's own map in every caller of
// the reference; candidates are filtered natively (keepAccelerator rule, server.go:70-82).
func (s *Server) Calculate(accelerators map[string]*Accelerator) {
	s.allAllocations = map[string]*Allocation{}
	if s.system == nil || s.system.analyzeAll() != nil {
		return
	}
	for name, ai := range s.system.accIndex {
		if _, listed := accelerators[name]; !listed {
			continue
		}
		if al := s.system.pairAllocation(s.index, ai, false); al != nil {
			s.allAllocations[name] = al
		}
	}
}
func (s *Server) Name() string                          { return s.name }
func (s *Server) ServiceClassName() string              { return s.serviceClassName }
func (s *Server) ModelName() string                     { return s.modelName }
func (s *Server) KeepAccelerator() bool                 { return s.keepAccelerator }
func (s *Server) Load() *config.ServerLoadSpec          { return s.load }
func (s *Server) SetLoad(l *config.ServerLoadSpec)      { s.load = l; s.invalidate() }
func (s *Server) Allocation() *Allocation               { return s.allocation }
func (s *Server) SetAllocation(a *Allocation)           { s.allocation = a; s.UpdateDesiredAlloc() }
func (s *Server) RemoveAllocation()                     { s.allocation = nil }
func (s *Server) CurAllocation() *Allocation            { return s.curAllocation }
func (s *Server) SetCurAllocation(a *Allocation)        { s.curAllocation = a; s.invalidate() }
func (s *Server) AllAllocations() map[string]*Allocation { return s.allAllocations }
func (s *Server) Spec() *config.ServerSpec              { return s.spec }
func (s *Server) Saturated() bool {
	return s.allocation != nil && s.load != nil && s.allocation.Saturated(s.load.ArrivalRate)
}
func (s *Server) Priority() int {
	if s.system != nil {
		if svc := s.system.serviceClasses[s.serviceClassName]; svc != nil {
			return svc.Priority()
		}
	}
	return config.DefaultServiceClassPriority
}
func (s *Server) UpdateDesiredAlloc() {
	if s.allocation != nil {
		s.spec.DesiredAlloc = *s.allocation.AllocationData()
		s.spec.DesiredAlloc.Load = *s.load
	} else {
		s.spec.DesiredAlloc = config.AllocationData{}
	}
}
func (s *Server) ApplyDesiredAlloc() {
	s.spec.CurrentAlloc = s.spec.DesiredAlloc
	s.curAllocation = AllocationFromData(&s.spec.CurrentAlloc)
	s.load = &s.spec.CurrentAlloc.Load
	s.invalidate()
}
func (s *Server) invalidate() {
	if s.system != nil {
		s.system.uploaded = false
	}
}

// ---- System (system.go) -----------------------------------------------------------------------------

type AllocationByType struct {
	name         string
	count, limit int
	cost         float32
}

func (a *AllocationByType) String() string {
	return fmt.Sprintf("name=%s, count=%d, limit=%d, cost=%v", a.name, a.count, a.limit, a.cost)
}

type System struct {
	accelerators   map[string]*Accelerator
	models         map[string]*Model
	serviceClasses map[string]*ServiceClass
	servers        map[string]*Server

	capacity           map[string]int
	allocationByType   map[string]*AllocationByType
	allocationSolution *config.AllocationSolution

	// native side
	ctx         *native.Context
	uploaded    bool
	analyzed    bool
	accNames    []string
	typeNames   []string
	serverNames []string
	accIndex    map[string]int
	serverIndex map[string]int
	image       *native.SystemImage
	pairs       *native.Allocs
	feasible    []uint8
	shared      map[int]*Allocation // pair index -> the one *Allocation handed out (the reference shares pointers)
}

func NewSystem() *System {
	return &System{accelerators: map[string]*Accelerator{}, models: map[string]*Model{},
		serviceClasses: map[string]*ServiceClass{}, servers: map[string]*Server{}, capacity: map[string]int{},
		allocationByType: map[string]*AllocationByType{}}
}

func (s *System) SetFromSpec(d *config.SystemSpec) *config.OptimizerSpec {
	for i := range d.Accelerators.Spec {
		s.AddAcceleratorFromSpec(d.Accelerators.Spec[i])
	}
	for i := range d.Models.PerfData {
		pd := &d.Models.PerfData[i]
		m := s.models[pd.Name]
		if m == nil {
			m = s.AddModel(pd.Name)
		}
		m.AddPerfDataFromSpec(pd)
	}
	for i := range d.ServiceClasses.Spec {
		s.serviceClasses[d.ServiceClasses.Spec[i].Name] = NewServiceClassFromSpec(&d.ServiceClasses.Spec[i])
	}
	for i := range d.Servers.Spec {
		s.AddServerFromSpec(d.Servers.Spec[i])
	}
	for _, c := range d.Capacity.Count {
		s.capacity[c.Type] = c.Count
	}
	s.uploaded = false
	return &d.Optimizer.Spec
}
func (s *System) AddAcceleratorFromSpec(spec config.AcceleratorSpec) {
	s.accelerators[spec.Name] = NewAcceleratorFromSpec(&spec)
	s.uploaded = false
}
func (s *System) AddModel(name string) *Model { m := NewModel(name); s.models[name] = m; s.uploaded = false; return m }
func (s *System) AddServerFromSpec(spec config.ServerSpec) {
	sv := NewServerFromSpec(&spec)
	sv.system = s
	s.servers[spec.Name] = sv
	s.uploaded = false
}
func (s *System) AddServiceClass(name string, priority int) { s.serviceClasses[name] = NewServiceClass(name, priority); s.uploaded = false }
func (s *System) SetCountFromSpec(spec config.AcceleratorCount) { s.capacity[spec.Type] = spec.Count; s.uploaded = false }
func (s *System) RemoveServer(name string) error {
	if s.servers[name] == nil {
		return fmt.Errorf("server %s not found", name)
	}
	delete(s.servers, name)
	s.uploaded = false
	return nil
}
func (s *System) Accelerators() map[string]*Accelerator     { return s.accelerators }
func (s *System) Models() map[string]*Model                 { return s.models }
func (s *System) ServiceClasses() map[string]*ServiceClass  { return s.serviceClasses }
func (s *System) Servers() map[string]*Server               { return s.servers }
func (s *System) Accelerator(n string) *Accelerator         { return s.accelerators[n] }
func (s *System) Model(n string) *Model                     { return s.models[n] }
func (s *System) ServiceClass(n string) *ServiceClass       { return s.serviceClasses[n] }
func (s *System) Server(n string) *Server                   { return s.servers[n] }
func (s *System) Capacities() map[string]int                { return s.capacity }
func (s *System) Capacity(n string) (int, bool)             { c, ok := s.capacity[n]; return c, ok }

// Calculate (system.go:262-272)
func (s *System) Calculate() {
	// callers may have mutated loads / specs through the shared pointers (server.Load(), Spec()): the image is
	// rebuilt and re-sent on every Calculate (51 MB at 100 000 servers x 16 accelerators)
	s.uploaded = false
	for _, v := range s.servers {
		v.Calculate(s.accelerators)
	}
}

// upload builds the structure-of-arrays image (string interning, class/target resolution) and sends it.
func (s *System) upload() error {
	if s.uploaded {
		return nil
	}
	if s.ctx == nil {
		c, err := native.Default()
		if err != nil {
			return err
		}
		s.ctx = c
	}
	img := &native.SystemImage{}
	s.accNames, s.typeNames, s.serverNames = s.accNames[:0], s.typeNames[:0], s.serverNames[:0]
	s.accIndex, s.serverIndex = map[string]int{}, map[string]int{}
	typeIndex, modelIndex := map[string]int{}, map[string]int{}
	for _, n := range sortedKeys(s.accelerators) {
		s.accIndex[n] = len(s.accNames)
		s.accNames = append(s.accNames, n)
		t := s.accelerators[n].Type()
		if _, ok := typeIndex[t]; !ok {
			typeIndex[t] = len(s.typeNames)
			s.typeNames = append(s.typeNames, t)
		}
	}
	modelNames := sortedKeys(s.models)
	for i, n := range modelNames {
		modelIndex[n] = i
	}
	for _, n := range sortedKeys(s.servers) {
		s.serverIndex[n] = len(s.serverNames)
		s.serverNames = append(s.serverNames, n)
		s.servers[n].index = s.serverIndex[n]
		s.servers[n].system = s
	}
	S, A, M, T := len(s.serverNames), len(s.accNames), len(modelNames), len(s.typeNames)
	img.S, img.A, img.M, img.T = S, A, M, T
	img.AccCost, img.AccMultiplicity, img.AccType = make([]float32, A), make([]int32, A), make([]int32, A)
	img.TypeCapacity = make([]int64, T)
	for i, n := range s.accNames {
		g := s.accelerators[n]
		img.AccCost[i], img.AccMultiplicity[i], img.AccType[i] = g.Cost(), int32(g.Multiplicity()), int32(typeIndex[g.Type()])
	}
	for i, t := range s.typeNames {
		img.TypeCapacity[i] = int64(s.capacity[t])
	}
	MA := M * A
	img.PerfAlpha, img.PerfBeta, img.PerfGamma, img.PerfDelta = make([]float32, MA), make([]float32, MA), make([]float32, MA), make([]float32, MA)
	img.PerfMaxBatch, img.PerfAtTokens, img.PerfAccCount, img.PerfValid = make([]int32, MA), make([]int32, MA), make([]int32, MA), make([]uint8, MA)
	for mi, mn := range modelNames {
		for an, pd := range s.models[mn].perfData {
			ai, ok := s.accIndex[an]
			if !ok {
				continue
			}
			k := mi*A + ai
			img.PerfAlpha[k], img.PerfBeta[k] = pd.DecodeParms.Alpha, pd.DecodeParms.Beta
			img.PerfGamma[k], img.PerfDelta[k] = pd.PrefillParms.Gamma, pd.PrefillParms.Delta
			img.PerfMaxBatch[k], img.PerfAtTokens[k], img.PerfAccCount[k], img.PerfValid[k] = int32(pd.MaxBatchSize), int32(pd.AtTokens), int32(pd.AccCount), 1
		}
	}
	img.SrvModel, img.SrvArrivalRPM = make([]int32, S), make([]float32, S)
	img.SrvInTokens, img.SrvOutTokens = make([]int32, S), make([]int32, S)
	img.SrvSloTTFT, img.SrvSloITL, img.SrvSloTPS, img.SrvTargetValid = make([]float32, S), make([]float32, S), make([]float32, S), make([]uint8, S)
	img.SrvPriority, img.SrvMinReplicas, img.SrvMaxBatch, img.SrvKeepAcc = make([]int32, S), make([]int32, S), make([]int32, S), make([]uint8, S)
	img.SrvCurAcc, img.SrvCurReplicas, img.SrvCurCost = make([]int32, S), make([]int32, S), make([]float32, S)
	for i, n := range s.serverNames {
		sv := s.servers[n]
		img.SrvModel[i] = -1
		if mi, ok := modelIndex[sv.modelName]; ok {
			img.SrvModel[i] = int32(mi)
		}
		if sv.load != nil {
			img.SrvArrivalRPM[i], img.SrvInTokens[i], img.SrvOutTokens[i] = sv.load.ArrivalRate, int32(sv.load.AvgInTokens), int32(sv.load.AvgOutTokens)
		} else {
			img.SrvArrivalRPM[i] = -1 // load == nil => CreateAllocation returns nil (allocation.go:49-52)
		}
		img.SrvPriority[i] = int32(sv.Priority())
		if svc := s.serviceClasses[sv.serviceClassName]; svc != nil {
			if t := svc.ModelTarget(sv.modelName); t != nil {
				img.SrvTargetValid[i], img.SrvSloITL[i], img.SrvSloTTFT[i], img.SrvSloTPS[i] = 1, t.ITL, t.TTFT, t.TPS
			}
		}
		img.SrvMinReplicas[i], img.SrvMaxBatch[i] = int32(sv.minNumReplicas), int32(sv.maxBatchSize)
		if sv.keepAccelerator {
			img.SrvKeepAcc[i] = 1
		}
		img.SrvCurAcc[i] = -1 // WVA_ACC_NONE
		if cur := sv.curAllocation; cur != nil {
			if cur.accelerator != "" {
				if ai, ok := s.accIndex[cur.accelerator]; ok {
					img.SrvCurAcc[i] = int32(ai)
				} else {
					img.SrvCurAcc[i] = -2 // WVA_ACC_UNKNOWN
				}
			}
			img.SrvCurReplicas[i], img.SrvCurCost[i] = int32(cur.numReplicas), cur.cost
		}
	}
	if err := s.ctx.Upload(img); err != nil {
		return err
	}
	s.image, s.uploaded, s.analyzed = img, true, false
	return nil
}

func (s *System) analyzeAll() error {
	if err := s.upload(); err != nil {
		return err
	}
	if s.analyzed {
		return nil
	}
	pairs, fe, err := s.ctx.AnalyzePairs(s.image.S, s.image.A)
	if err != nil {
		return err
	}
	s.pairs, s.feasible, s.analyzed, s.shared = pairs, fe, true, map[int]*Allocation{}
	return nil
}

func (s *System) allocFromRecord(r *native.Allocs, i int) *Allocation {
	name := ""
	if r.Acc[i] >= 0 {
		name = s.accNames[r.Acc[i]]
	}
	return &Allocation{accelerator: name, numReplicas: int(r.NumReplicas[i]), batchSize: int(r.BatchSize[i]), cost: r.Cost[i],
		value: r.Value[i], itl: r.ITL[i], ttft: r.TTFT[i], rho: r.Rho[i], maxArrvRatePerReplica: r.MaxArrv[i]}
}

// pairAllocation returns the allocation of (server si, accelerator ai) or nil; fresh = a private copy.
func (s *System) pairAllocation(si, ai int, fresh bool) *Allocation {
	i := si*s.image.A + ai
	if s.feasible == nil || s.feasible[i] == 0 {
		return nil
	}
	if fresh {
		return s.allocFromRecord(s.pairs, i)
	}
	if al := s.shared[i]; al != nil {
		return al
	}
	al := s.allocFromRecord(s.pairs, i)
	s.shared[i] = al
	return al
}

// Solve is called by solver.Solver: runs the assignment natively and installs server.allocation.
func (s *System) Solve(spec *config.OptimizerSpec) (solutionTimeUsec int64, err error) {
	if err = s.analyzeAll(); err != nil {
		return 0, err
	}
	key, chosen, usec, err := s.ctx.Solve(s.image.S, spec.Unlimited, spec.DelayedBestEffort,
		int(config.SaturatedAllocationPolicyEnum(spec.SaturationPolicy)))
	if err != nil {
		return 0, err
	}
	for i, n := range s.serverNames {
		sv := s.servers[n]
		sv.RemoveAllocation()
		if key[i] < 0 {
			continue
		}
		al := s.pairAllocation(i, int(key[i]), false)
		if al == nil {
			al = &Allocation{}
		}
		// best-effort policies scale cost/value/replicas of the shared record in place (greedy.go:208-212)
		*al = *s.allocFromRecord(chosen, i)
		if sv.allAllocations != nil {
			sv.allAllocations[s.accNames[key[i]]] = al
		}
		sv.SetAllocation(al)
	}
	if !spec.Unlimited {
		s.analyzed = false // the device copy of the candidates was consumed
	}
	return usec, nil
}

// SolveAtCapacities runs the limited solve of spec under each of nVec capacity vectors (capacity[j*T+t]: vector j's count
// of the t-th accelerator type of the uploaded image) in one native call.  Server allocations, the candidates and the
// system's capacities are left as they were.
func (s *System) SolveAtCapacities(spec *config.OptimizerSpec, capacity []int64, nVec int) (*native.CapacityScenarios, error) {
	if err := s.analyzeAll(); err != nil {
		return nil, err
	}
	return s.ctx.SolveAtCapacities(capacity, nVec, spec.DelayedBestEffort, int(config.SaturatedAllocationPolicyEnum(spec.SaturationPolicy)))
}

// SolveAtArrivalRates runs the limited solve of spec under each of nLoads arrival-rate scenarios (rpm[srv*nLoads+j]:
// server srv's ArrivalRate in req/min in scenario j, servers in the uploaded image's order) on the system's capacities in
// one native call.  Server allocations, loads, candidates and capacities are left as they were.
func (s *System) SolveAtArrivalRates(spec *config.OptimizerSpec, rpm []float32, nLoads int) (*native.CapacityScenarios, error) {
	if err := s.upload(); err != nil {
		return nil, err
	}
	return s.ctx.SolveAtArrivalRates(rpm, nLoads, spec.DelayedBestEffort, int(config.SaturatedAllocationPolicyEnum(spec.SaturationPolicy)))
}

// AllocateByType (system.go:271-300)
func (s *System) AllocateByType() {
	s.allocationByType = map[string]*AllocationByType{}
	if s.image == nil {
		return
	}
	count, cost, err := s.ctx.AllocateByType(s.image.T)
	if err != nil {
		return
	}
	for _, sv := range s.servers {
		al := sv.Allocation()
		if al == nil {
			continue
		}
		acc := s.accelerators[al.accelerator]
		if acc == nil || s.models[sv.modelName] == nil {
			continue
		}
		t := acc.Type()
		if _, ok := s.allocationByType[t]; ok {
			continue
		}
		for ti, tn := range s.typeNames {
			if tn == t {
				s.allocationByType[t] = &AllocationByType{name: t, count: int(count[ti]), limit: s.capacity[t], cost: cost[ti]}
			}
		}
	}
}

// GenerateSolution (system.go:303-319)
func (s *System) GenerateSolution() *config.AllocationSolution {
	sol := config.AllocationSolution{Spec: map[string]config.AllocationData{}}
	for name, sv := range s.servers {
		al := sv.Allocation()
		if al == nil {
			continue
		}
		d := al.AllocationData()
		d.Load = *sv.Load()
		sol.Spec[name] = *d
	}
	s.allocationSolution = &sol
	return &sol
}
