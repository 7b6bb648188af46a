//! Lowering of `LookupAir::eval` to the backend's lookup program (`mdn_air.lookup`, include/miden_b200.h), so that the
//! LogUp aux trace -- `build_logup_aux_trace`, air/src/lookup/aux_builder.rs:49-97 -- is built ON THE DEVICE from the
//! main trace that is already resident in HBM: no host aux build between the main and aux commitments, no aux upload.
//!
//! The recording builder below is the symbolic twin of the reference's two adapters:
//!   * like `ConstraintLookupBuilder` (air/src/lookup/constraint.rs) it runs over the p3 symbolic types, so every flag,
//!     multiplicity and encoded message is an expression tree over main / preprocessed / periodic / public leaves and
//!     the two challenges alpha = CHALLENGE(0), beta = CHALLENGE(1) (`Challenges::new`, air/src/lookup/challenges.rs);
//!     a `CombinedWindow` read of the preprocessed part lowers to PREPROCESSED(offset, column) (op 15);
//!   * like `ProverLookupBuilder` (air/src/lookup/prover.rs:230-444) it keeps one record per interaction -- the
//!     `(multiplicity, encoded denominator)` pair the prover path pushes when the (boolean) flag is set -- instead of
//!     folding them into the `(V, U)` constraint pair, and it runs only the `canonical` closure of
//!     `group_with_cached_encoding`.
//! Record: `{aux column, flag node | 0xFFFFFFFF, multiplicity node, denominator node}`; on the device a row contributes
//! multiplicity / denominator to its column wherever the flag is non-zero (prover.rs:338-362), the fraction columns
//! c > 0 hold the per-row sums, column 0 the running sum, and the committed final is the grand total
//! (aux_builder.rs:1-20, 215-268).
//!
//! NOT COMPILED in this repository (no Rust toolchain in the build image); written against the sources as read.

use miden_air::lookup::{Challenges, Deg, LookupAir, LookupBatch, LookupBuilder, LookupColumn, LookupGroup, LookupMessage};
use miden_core::{Felt, field::{PrimeCharacteristicRing, QuadFelt}};   // PrimeCharacteristicRing: Felt::ONE
use miden_crypto::stark::air::{
    AirBuilder, ExtensionBuilder, PermutationAirBuilder,   // PermutationAirBuilder: permutation_randomness()
    symbolic::{AirLayout, SymbolicAirBuilder, SymbolicExpression, SymbolicExpressionExt},
};

use crate::lower::{Lowerer, MAGIC_LOOKUP, OpList};

type SB = SymbolicAirBuilder<Felt, QuadFelt>;
type Expr = SymbolicExpression<Felt>;
type ExprEF = SymbolicExpressionExt<Felt, QuadFelt>;

/// One `LookupGroup::insert` / `LookupBatch::insert` after `LookupMessage::encode`.
struct Interaction {
    column: u32,
    flag: Option<Expr>,
    multiplicity: Expr,
    denominator: ExprEF,
}

/// `LookupBuilder` over the symbolic AIR builder that records interactions.
pub struct RecordingLookupBuilder {
    sb: SB,
    challenges: Challenges<ExprEF>,
    column_idx: u32,
    interactions: Vec<Interaction>,
}

impl RecordingLookupBuilder {
    /// `layout` is the AIR's `air_layout()` (crates/lifted-air/src/air.rs:101-113): it fixes the main width, the
    /// periodic columns and the two LogUp challenges the expressions may refer to.
    pub fn new<A: LookupAir<Self>>(layout: AirLayout, air: &A) -> Self {
        let sb = SB::new(layout);
        let (alpha, beta): (ExprEF, ExprEF) = {
            let r = sb.permutation_randomness(); // constraint.rs:57-61
            (r[0].into(), r[1].into())
        };
        let challenges = Challenges::<ExprEF>::new(alpha, beta, air.max_message_width(), air.num_bus_ids());
        Self { sb, challenges, column_idx: 0, interactions: Vec::new() }
    }

    /// Serialise the recorded interactions as a lookup program.  `num_columns` = `LookupAir::num_columns()`.
    pub fn into_program(self, num_columns: usize) -> Vec<u32> {
        assert_eq!(self.column_idx as usize, num_columns, "LookupAir opened a different number of columns than it declares");
        let mut ops = OpList::default();
        let mut items = Vec::with_capacity(4 * self.interactions.len());
        {
            let mut lw = Lowerer::new(&mut ops);
            for it in &self.interactions {
                let flag = match &it.flag {
                    None => u32::MAX,
                    Some(f) => lw.base(f),
                };
                let mult = lw.base(&it.multiplicity);
                let den = lw.ext(&it.denominator);
                items.extend_from_slice(&[it.column, flag, mult, den]);
            }
        }
        ops.serialize(MAGIC_LOOKUP, &items, 4)
    }
}

/// A literal one needs no flag node.
fn flag_of(flag: Expr) -> Option<Expr> {
    match &flag {
        SymbolicExpression::Leaf(miden_crypto::stark::air::symbolic::BaseLeaf::Constant(c)) if *c == Felt::ONE => None,
        _ => Some(flag),
    }
}

impl LookupBuilder for RecordingLookupBuilder {
    type F = Felt;
    type Expr = Expr;
    type Var = <SB as AirBuilder>::Var;
    type EF = QuadFelt;
    type ExprEF = ExprEF;
    type VarEF = <SB as ExtensionBuilder>::VarEF;
    type PeriodicVar = <SB as AirBuilder>::PeriodicVar;
    type MainWindow = <SB as AirBuilder>::MainWindow;
    type Column<'a>
        = RecordingColumn<'a>
    where
        Self: 'a;

    fn main(&self) -> Self::MainWindow {
        self.sb.main()
    }
    fn periodic_values(&self) -> &[Self::PeriodicVar] {
        self.sb.periodic_values()
    }
    fn next_column<'a, R>(&'a mut self, f: impl FnOnce(&mut Self::Column<'a>) -> R, _deg: Deg) -> R {
        let column = self.column_idx;
        self.column_idx += 1;
        let mut col = RecordingColumn { challenges: &self.challenges, out: &mut self.interactions, column };
        f(&mut col)
    }
}

pub struct RecordingColumn<'c> {
    challenges: &'c Challenges<ExprEF>,
    out: &'c mut Vec<Interaction>,
    column: u32,
}

impl<'c> LookupColumn for RecordingColumn<'c> {
    type Expr = Expr;
    type ExprEF = ExprEF;
    type Group<'g>
        = RecordingGroup<'g>
    where
        Self: 'g;

    fn group<'g>(&'g mut self, _name: &'static str, f: impl FnOnce(&mut Self::Group<'g>), _deg: Deg) {
        let mut g = RecordingGroup { challenges: self.challenges, out: &mut *self.out, column: self.column };
        f(&mut g)
    }
    fn group_with_cached_encoding<'g>(
        &'g mut self,
        name: &'static str,
        canonical: impl FnOnce(&mut Self::Group<'g>),
        _encoded: impl FnOnce(&mut Self::Group<'g>),
        deg: Deg,
    ) {
        // prover semantics: the canonical closure only (prover.rs:283-293)
        self.group(name, canonical, deg);
    }
}

pub struct RecordingGroup<'g> {
    challenges: &'g Challenges<ExprEF>,
    out: &'g mut Vec<Interaction>,
    column: u32,
}

impl<'g> LookupGroup for RecordingGroup<'g> {
    type Expr = Expr;
    type ExprEF = ExprEF;
    type Batch<'b>
        = RecordingBatch<'b>
    where
        Self: 'b;

    fn insert<M>(&mut self, _name: &'static str, flag: Expr, multiplicity: Expr, msg: impl FnOnce() -> M, _deg: Deg)
    where
        M: LookupMessage<Expr, ExprEF>,
    {
        let denominator = msg().encode(self.challenges);
        self.out.push(Interaction { column: self.column, flag: flag_of(flag), multiplicity, denominator });
    }
    fn batch<'b>(&'b mut self, _name: &'static str, flag: Expr, build: impl FnOnce(&mut Self::Batch<'b>), _deg: Deg) {
        let mut b = RecordingBatch { challenges: self.challenges, out: &mut *self.out, column: self.column, flag: flag_of(flag) };
        build(&mut b)
    }
}

pub struct RecordingBatch<'b> {
    challenges: &'b Challenges<ExprEF>,
    out: &'b mut Vec<Interaction>,
    column: u32,
    flag: Option<Expr>,
}

impl<'b> LookupBatch for RecordingBatch<'b> {
    type Expr = Expr;
    type ExprEF = ExprEF;

    fn insert<M>(&mut self, _name: &'static str, multiplicity: Expr, msg: M, _deg: Deg)
    where
        M: LookupMessage<Expr, ExprEF>,
    {
        let denominator = msg.encode(self.challenges);
        self.out.push(Interaction { column: self.column, flag: self.flag.clone(), multiplicity, denominator });
    }
    fn insert_encoded(&mut self, _name: &'static str, multiplicity: Expr, encoded: impl FnOnce() -> ExprEF, _deg: Deg) {
        self.out.push(Interaction { column: self.column, flag: self.flag.clone(), multiplicity, denominator: encoded() });
    }
}

/// Lower the `LookupAir` of one AIR: `(num_columns, program words)` for `mdn_lookup`.
/// The backend requires `aux_width == num_columns` (<= 16) and `num_aux_values == 1` -- the shape of every AIR whose
/// `build_aux_trace` is `build_logup_aux_trace` (all three Miden AIRs, air/src/lib.rs:273-274, 671-685).
/// This emits version-1 programs only.  AIRs whose aux trace is a LogUp trace followed by register columns (the uint
/// chiplets' Schwartz-Zippel columns, precompiles-prover/src/uint/trace.rs) need a version-2 program: one update node
/// per register after the interactions, AUX(0, num_columns + i) for register i's row value, every update affine in
/// the registers (include/miden_b200.h `mdn_lookup`).  The recorder does not capture those updates yet.
pub fn lower_lookup<A>(layout: AirLayout, air: &A) -> (u32, Vec<u32>)
where
    A: LookupAir<RecordingLookupBuilder>,
{
    let mut b = RecordingLookupBuilder::new(layout, air);
    air.eval(&mut b);
    let n = air.num_columns();
    (n as u32, b.into_program(n))
}
