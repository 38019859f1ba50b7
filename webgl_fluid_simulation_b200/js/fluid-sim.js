// fluid-sim.js — the reference's simulation surface in its own language, over the N-API shim.
//
// The host-side helpers below (pointerPrototype, HSVtoRGB, wrap, generateColor, multipleSplats,
// splatPointer, calcDeltaTime, updateColors, applyInputs, updatePointer*Data, correctDelta*) keep
// the names, argument order and arithmetic of PavelDoGreat/WebGL-Fluid-Simulation's script.js so
// that this module is a drop-in for its simulation path; those parts are
//     Copyright (c) 2017 Pavel Dobryakov, MIT License (see LICENSE at the repository root).
// No shader / compute code of the reference is reproduced: all simulation work happens in
// libfluid_b200 (hand-written CUDA).
//
// NOT EXECUTED IN THIS REPOSITORY: the build image has no Node (`node --version`: not found) and
// no browser, so this file is the integration artefact for a maintainer, kept in lock-step with
// its tested Python twin webgl_fluid_simulation_b200/sim.py (same structure, same names).
//
// It keeps the names and semantics of script.js ("S"): `config` (S:59-85), `step(dt)`
// (S:1231-1294), `splat(x, y, dx, dy, color)` (S:1441-1455), `multipleSplats(amount)`
// (S:1427-1439), `splatPointer(pointer)` (S:1421-1425), `initFramebuffers()` (S:982-1010),
// `generateColor()` (S:1565-1571), `calcDeltaTime()` (S:1188-1194), `update()` (S:1176-1186),
// `pointers` / `splatStack` (S:87-102), and the field objects `velocity / dye / pressure /
// divergence / curl` (S:950-954) whose `.read()` returns a Float32Array where the reference
// would bind a texture.  `config` is read live on every call, like the reference does.
'use strict';

const native = require('../napi/fluid.node');

const FIELD = { velocity: 0, dye: 1, pressure: 2, divergence: 3, curl: 4 };
const PARAM = {
    DENSITY_DISSIPATION: 0, VELOCITY_DISSIPATION: 1, PRESSURE: 2, PRESSURE_ITERATIONS: 3,
    CURL: 4, SPLAT_RADIUS: 5, ASPECT: 6, JACOBI_BLOCK: 7, BACKGROUND: 8,
};
// display keywords of render() (updateKeywords, S:1160-1166): FLUID_DISPLAY_* of include/fluid.h
const DISPLAY = { SHADING: 0x1, BLOOM: 0x2, SUNRAYS: 0x4 };
const FLAG = { UNFUSED: 0x1, NO_GRAPH: 0x2, NAIVE_JACOBI: 0x4, TILED_PASSES: 0x8, HALF_STORAGE: 0x10, HALF_POSTFX: 0x20,
               NEAREST_FILTERING: 0x40, LINEAR_ADVECTION: 0x80 };
const STAT = { launches: 0, jacobiLaunches: 1, haloLaunches: 2, haloExchanges: 3, graphCaptures: 4, graphLaunches: 5, haloTransportP2P: 6,
               cvdStreamLaunches: 7, gradientStreamLaunches: 8, jacobiExactStreams: 9, advect4Launches: 10, gathers: 11 };

function pointerPrototype () {                                  // S:87-98
    this.id = -1;
    this.texcoordX = 0;
    this.texcoordY = 0;
    this.prevTexcoordX = 0;
    this.prevTexcoordY = 0;
    this.deltaX = 0;
    this.deltaY = 0;
    this.down = false;
    this.moved = false;
    this.color = { r: 30, g: 0, b: 300 };                       // an {r,g,b} object like generateColor() returns (splat reads .r/.g/.b)
}

function HSVtoRGB (h, s, v) {                                   // S:1573-1597
    let r, g, b;
    const i = Math.floor(h * 6);
    const f = h * 6 - i;
    const p = v * (1 - s);
    const q = v * (1 - f * s);
    const t = v * (1 - (1 - f) * s);
    switch (i % 6) {
        case 0: r = v; g = t; b = p; break;
        case 1: r = q; g = v; b = p; break;
        case 2: r = p; g = v; b = t; break;
        case 3: r = p; g = q; b = v; break;
        case 4: r = t; g = p; b = v; break;
        case 5: r = v; g = p; b = q; break;
    }
    return { r, g, b };
}

function wrap (value, min, max) {                               // S:1599-1603
    const range = max - min;
    if (range == 0) return min;
    return (value - min) % range + min;
}

class FluidSimulation {
    constructor (config = {}, canvas = { width: 1024, height: 1024 }, options = {}) {
        this.config = Object.assign({                           // S:59-85
            SIM_RESOLUTION: 128,
            DYE_RESOLUTION: 1024,
            CAPTURE_RESOLUTION: 512,    // S:62
            DENSITY_DISSIPATION: 1,
            VELOCITY_DISSIPATION: 0.2,
            PRESSURE: 0.8,
            PRESSURE_ITERATIONS: 20,
            CURL: 30,
            SPLAT_RADIUS: 0.25,
            SPLAT_FORCE: 6000,
            SHADING: true,
            COLORFUL: true,
            COLOR_UPDATE_SPEED: 10,
            PAUSED: false,
            BACK_COLOR: { r: 0, g: 0, b: 0 },
            TRANSPARENT: false,
            BLOOM: false,           // reference default is true; needs `sim.dithering` (the 64x64 RGB texture), see render()
            BLOOM_ITERATIONS: 8,
            BLOOM_RESOLUTION: 256,
            BLOOM_INTENSITY: 0.8,
            BLOOM_THRESHOLD: 0.6,
            BLOOM_SOFT_KNEE: 0.7,
            SUNRAYS: false,         // reference default is true
            SUNRAYS_RESOLUTION: 196,
            SUNRAYS_WEIGHT: 1.0,
        },
        // a device without float linear filtering (S:109-114); the caller's keys win, as later GUI edits do
        (options.flags || 0) & FLAG.NEAREST_FILTERING ? { DYE_RESOLUTION: 512, SHADING: false, BLOOM: false, SUNRAYS: false } : {},
        config);
        this.dithering = null;                                  // {width, height, data: Float32Array RGB}, LDR_LLL1_0.png / 255
        this.canvas = canvas;
        this.random = options.random || Math.random;            // injectable for reproducible runs
        this.options = options;
        this.pointers = [new pointerPrototype()];               // S:100-102
        this.splatStack = [];
        this.lastUpdateTime = Date.now();                       // S:1172
        this.colorUpdateTimer = 0.0;
        this._h = null;
        this._pushed = {};
        for (const name of Object.keys(FIELD)) {
            this[name] = {
                read: () => native.read(this._h, FIELD[name]),
                get width () { return native.dims(this._sim._h, FIELD[name]).width; },
                get height () { return native.dims(this._sim._h, FIELD[name]).height; },
                _sim: this,
            };
        }
        this.initFramebuffers();
    }

    _aspect () { return this.canvas.width / this.canvas.height; }

    _pushConfig () {                                            // config is read live (S:1243, S:1255, ...)
        const c = this.config;
        const vals = {
            DENSITY_DISSIPATION: c.DENSITY_DISSIPATION, VELOCITY_DISSIPATION: c.VELOCITY_DISSIPATION,
            PRESSURE: c.PRESSURE, PRESSURE_ITERATIONS: c.PRESSURE_ITERATIONS, CURL: c.CURL,
            SPLAT_RADIUS: c.SPLAT_RADIUS, ASPECT: this._aspect(),
        };
        for (const k of Object.keys(vals)) {
            if (this._pushed[k] !== vals[k]) {
                native.setParam(this._h, PARAM[k], vals[k]);
                this._pushed[k] = vals[k];
            }
        }
    }

    initFramebuffers () {                                       // S:982-1010
        const simRes = native.getResolution(this.config.SIM_RESOLUTION, this.canvas.width, this.canvas.height);
        const dyeRes = native.getResolution(this.config.DYE_RESOLUTION, this.canvas.width, this.canvas.height);
        if (this._h == null) {
            this._h = native.create(Object.assign({}, this.config, {
                simWidth: simRes.width, simHeight: simRes.height,
                dyeWidth: dyeRes.width, dyeHeight: dyeRes.height,
                aspect: this._aspect(), device: this.options.device === undefined ? -1 : this.options.device,
                flags: this.options.flags || 0, jacobiBlock: this.options.jacobiBlock || 0,
            }));
        } else {                                                // resizeDoubleFBO, S:1116-1126
            native.resize(this._h, simRes.width, simRes.height, dyeRes.width, dyeRes.height);
        }
        this._pushed = {};
        this._pushConfig();
    }

    step (dt) {                                                 // S:1231-1294
        this._pushConfig();
        native.step(this._h, dt);
    }

    splat (x, y, dx, dy, color) {                               // S:1441-1455
        this._pushConfig();
        native.splat(this._h, x, y, dx, dy, color.r, color.g, color.b);
    }

    // len/7 splat() calls in one: records is a Float32Array of (x, y, dx, dy, r, g, b) records,
    // applied in order with the same result as one splat() per record, in ceil(n/128) launches
    splats (records) {
        if (!(records instanceof Float32Array) || records.length % 7 !== 0)
            throw new TypeError('splats() takes a Float32Array of 7-float records (x, y, dx, dy, r, g, b)');
        this._pushConfig();
        native.splats(this._h, records);
    }

    splatPointer (pointer) {                                    // S:1421-1425
        const dx = pointer.deltaX * this.config.SPLAT_FORCE;
        const dy = pointer.deltaY * this.config.SPLAT_FORCE;
        this.splat(pointer.texcoordX, pointer.texcoordY, dx, dy, pointer.color);
    }

    multipleSplats (amount) {                                   // S:1427-1439
        for (let i = 0; i < amount; i++) {
            const color = this.generateColor();
            color.r *= 10.0;
            color.g *= 10.0;
            color.b *= 10.0;
            const x = this.random();
            const y = this.random();
            const dx = 1000 * (this.random() - 0.5);
            const dy = 1000 * (this.random() - 0.5);
            this.splat(x, y, dx, dy, color);
        }
    }

    generateColor () {                                          // S:1565-1571
        const c = HSVtoRGB(this.random(), 1.0, 1.0);
        c.r *= 0.15;
        c.g *= 0.15;
        c.b *= 0.15;
        return c;
    }

    calcDeltaTime () {                                          // S:1188-1194
        const now = Date.now();
        let dt = (now - this.lastUpdateTime) / 1000;
        dt = Math.min(dt, 0.016666);
        this.lastUpdateTime = now;
        return dt;
    }

    updateColors (dt) {                                         // S:1207-1217
        if (!this.config.COLORFUL) return;
        this.colorUpdateTimer += dt * this.config.COLOR_UPDATE_SPEED;
        if (this.colorUpdateTimer >= 1) {
            this.colorUpdateTimer = wrap(this.colorUpdateTimer, 0, 1);
            this.pointers.forEach(p => { p.color = this.generateColor(); });
        }
    }

    applyInputs () {                                            // S:1219-1229
        if (this.splatStack.length > 0) this.multipleSplats(this.splatStack.pop());
        this.pointers.forEach(p => {
            if (p.moved) {
                p.moved = false;
                this.splatPointer(p);
            }
        });
    }

    // S:1176-1186 minus rAF.  With draw = true it ends like the reference's, with render(null): the canvas
    // frame of renderCanvas() is returned (put it on the page with putImageData); otherwise dt.
    update (draw = false) {
        const dt = this.calcDeltaTime();
        this.updateColors(dt);
        this.applyInputs();
        if (!this.config.PAUSED) this.step(dt);
        return draw ? this.renderCanvas() : dt;
    }

    // ---- pointer helpers (the caller side of splat(); the DOM listeners S:1464-1525 stay with the page) ----
    updatePointerDownData (pointer, id, posX, posY) {           // S:1527-1538
        pointer.id = id;
        pointer.down = true;
        pointer.moved = false;
        pointer.texcoordX = posX / this.canvas.width;
        pointer.texcoordY = 1.0 - posY / this.canvas.height;
        pointer.prevTexcoordX = pointer.texcoordX;
        pointer.prevTexcoordY = pointer.texcoordY;
        pointer.deltaX = 0;
        pointer.deltaY = 0;
        pointer.color = this.generateColor();
    }

    updatePointerMoveData (pointer, posX, posY) {               // S:1540-1548
        pointer.prevTexcoordX = pointer.texcoordX;
        pointer.prevTexcoordY = pointer.texcoordY;
        pointer.texcoordX = posX / this.canvas.width;
        pointer.texcoordY = 1.0 - posY / this.canvas.height;
        pointer.deltaX = this.correctDeltaX(pointer.texcoordX - pointer.prevTexcoordX);
        pointer.deltaY = this.correctDeltaY(pointer.texcoordY - pointer.prevTexcoordY);
        pointer.moved = Math.abs(pointer.deltaX) > 0 || Math.abs(pointer.deltaY) > 0;
    }

    updatePointerUpData (pointer) { pointer.down = false; }     // S:1550-1552

    correctDeltaX (delta) {                                     // S:1554-1558
        const aspectRatio = this._aspect();
        if (aspectRatio < 1) delta *= aspectRatio;
        return delta;
    }

    correctDeltaY (delta) {                                     // S:1560-1564
        const aspectRatio = this._aspect();
        if (aspectRatio > 1) delta /= aspectRatio;
        return delta;
    }

    // render(target) of S:1296-1317: Float32Array RGBA, row 0 = bottom.  config.SHADING / BLOOM / SUNRAYS
    // pick the display keywords like updateKeywords (S:1160-1166); BLOOM needs this.dithering, BLOOM or
    // SUNRAYS a single-GPU fp32 handle.  config.TRANSPARENT: the checkerboard under the display on the
    // screen (target = false, S:1311-1312), the bare display into a capture target (target = true).
    render (width = this.canvas.width, height = this.canvas.height, target = false) {
        const c = this.config;
        const bc = c.BACK_COLOR;                                // normalizeColor, S:1599-1606
        const bg = !c.TRANSPARENT ? 0 : (target ? 2 : 1);
        if (this._pushed.BACKGROUND !== bg) {
            native.setParam(this._h, PARAM.BACKGROUND, bg);
            this._pushed.BACKGROUND = bg;
        }
        this._pushConfig();                                     // the checkerboard uses canvas.width / canvas.height (S:1327)
        const kw = this._keywords();
        const d = this.dithering;
        return native.renderKeywords(this._h, width, height, kw, c, (kw & DISPLAY.BLOOM) ? d.data : null,
                                     d ? d.width : 0, d ? d.height : 0, bc.r / 255, bc.g / 255, bc.b / 255);
    }

    // updateKeywords (S:1160-1166) as DISPLAY bits; BLOOM needs this.dithering
    _keywords () {
        const c = this.config;
        const kw = (c.SHADING ? DISPLAY.SHADING : 0) | (c.BLOOM ? DISPLAY.BLOOM : 0) | (c.SUNRAYS ? DISPLAY.SUNRAYS : 0);
        if ((kw & DISPLAY.BLOOM) && this.dithering == null)
            throw new Error('BLOOM needs sim.dithering: {width, height, data} of the 64x64 RGB dithering texture (LDR_LLL1_0.png / 255)');
        return kw;
    }

    // captureScreenshot() of S:287-299 up to normalizeTexture (S:309-327): render() into an RGBA half-float
    // target of getResolution(CAPTURE_RESOLUTION), quantised to 8 bits on the GPU.  The bloom and sunrays
    // FBOs keep the canvas sizes; TRANSPARENT stores the display bare.  Returns {width, height, data:
    // Uint8Array RGBA, top row first}: what textureToCanvas puts on the capture canvas.  toDataURL and the
    // download (S:296-298) stay in the page.
    captureScreenshot () {
        const c = this.config;
        const bc = c.BACK_COLOR;                                // normalizeColor, S:1599-1606
        const res = native.getResolution(c.CAPTURE_RESOLUTION, this.canvas.width, this.canvas.height);
        const kw = this._keywords();
        const d = this.dithering;
        const data = native.capture(this._h, res.width, res.height, this.canvas.width, this.canvas.height, kw,
                                    !!c.TRANSPARENT, c, (kw & DISPLAY.BLOOM) ? d.data : null, d ? d.width : 0,
                                    d ? d.height : 0, bc.r / 255, bc.g / 255, bc.b / 255);
        return { width: res.width, height: res.height, data };
    }

    // render(null) of S:1296-1317 on the canvas's RGBA8 drawing buffer (fluid_render_canvas in
    // include/fluid.h states the rule): canvas.width x canvas.height, the display over BACK_COLOR or, with
    // TRANSPARENT, the checkerboard, clamped and quantised like the fixed-point buffer.  Returns {width, height,
    // data: Uint8ClampedArray RGBA, top row first}: new ImageData(data, width, height) for ctx.putImageData.
    renderCanvas () {
        const c = this.config;
        const bc = c.BACK_COLOR;                                // normalizeColor, S:1599-1606
        this._pushConfig();                                     // the checkerboard uses canvas.width / canvas.height (S:1327)
        const kw = this._keywords();
        const d = this.dithering;
        const data = native.renderCanvas(this._h, this.canvas.width, this.canvas.height, kw, !!c.TRANSPARENT, c,
                                         (kw & DISPLAY.BLOOM) ? d.data : null, d ? d.width : 0, d ? d.height : 0,
                                         bc.r / 255, bc.g / 255, bc.b / 255);
        return { width: this.canvas.width, height: this.canvas.height, data };
    }

    stat (name) { return native.stat(this._h, STAT[name]); }
    destroy () { if (this._h != null) { native.destroy(this._h); this._h = null; } }   // frees device memory now, not at GC
    readField (name) { return native.read(this._h, FIELD[name]); }
    writeField (name, f32) { native.write(this._h, FIELD[name], f32); }
    sync () { native.sync(this._h); }
}

module.exports = { FluidSimulation, pointerPrototype, HSVtoRGB, wrap, FIELD, PARAM, DISPLAY, FLAG, STAT };
